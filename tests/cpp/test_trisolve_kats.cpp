// test_trisolve_kats.cpp -- the reference's trisolve tests (sprs/src/sparse/linalg/
// trisolve.rs:368-442) replayed through the C++ host mirror (include/sprs_b200.hpp) on the GPU,
// with the panics and a singular matrix.  Built and run by
// tests/test_gpu_trisolve.py::test_cpp_trisolve_kats (and on the emulator by
// tests/test_emu_trisolve.py); exits non-zero on the first failure.
#include <cstdio>
#include <cstdlib>

#include "../../include/sprs_b200.hpp"

using namespace sprs;
using namespace sprs::linalg;
static int g_checks = 0;
#define CHECK(cond)                                                             \
    do {                                                                        \
        ++g_checks;                                                             \
        if (!(cond)) {                                                          \
            fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);    \
            exit(1);                                                            \
        }                                                                       \
    } while (0)

template <class F>
static bool panics_with(F f, const char* msg) {
    try {
        f();
    } catch (const Panic& p) {
        return std::string(p.what()) == msg;
    }
    return false;
}

int main() {
    const Array1 want = {3., 1., 1.};
    // trisolve.rs:368-384
    const CsMat l = CsMat::new_({3, 3}, {0, 1, 2, 4}, {0, 1, 0, 2}, {1., 2., 1., 1.});
    Array1 x = {3., 2., 4.};
    trisolve::lsolve_csr_dense_rhs(l, x);
    CHECK(x == want);
    // trisolve.rs:386-406
    const CsMat lc = CsMat::new_csc({3, 3}, {0, 2, 3, 4}, {0, 1, 1, 2}, {1., 1., 2., 3.});
    x = {3., 5., 3.};
    trisolve::lsolve_csc_dense_rhs(lc, x);
    CHECK(x == want);
    // trisolve.rs:408-424
    const CsMat uc = CsMat::new_csc({3, 3}, {0, 1, 2, 4}, {0, 1, 0, 2}, {1., 2., 1., 3.});
    x = {4., 2., 3.};
    trisolve::usolve_csc_dense_rhs(uc, x);
    CHECK(x == want);
    // trisolve.rs:426-442
    const CsMat u = CsMat::new_({3, 3}, {0, 2, 4, 5}, {0, 1, 1, 2, 2}, {1., 1., 5., 3., 1.});
    x = {4., 8., 1.};
    trisolve::usolve_csr_dense_rhs(u, x);
    CHECK(x == want);
    // the panics, in the reference's order: square, rhs.dim(), storage
    const CsMat rect = CsMat::new_({2, 3}, {0, 1, 2}, {0, 1}, {1., 1.});
    Array1 bad(5);
    CHECK(panics_with([&] { trisolve::lsolve_csc_dense_rhs(rect, bad); },
                      "Non square matrix passed to solver"));
    CHECK(panics_with([&] { trisolve::lsolve_csc_dense_rhs(l, bad); }, "Dimension mismatch"));
    x = {3., 2., 4.};
    CHECK(panics_with([&] { trisolve::lsolve_csc_dense_rhs(l, x); }, "Storage mismatch"));
    // a structural 0 at column 1 of a CSC lower solve: column 0 applied, nothing divided
    const CsMat s = CsMat::new_csc({3, 3}, {0, 3, 4, 5}, {0, 1, 2, 2, 2}, {2., 1., 4., 3., 1.});
    x = {4., 5., 7.};
    bool thrown = false;
    try {
        trisolve::lsolve_csc_dense_rhs(s, x);
    } catch (const SingularMatrix& e) {
        thrown = e.index == 1 && e.reason == "diagonal element is a structural 0" &&
                 std::string(e.what()) == "Singular matrix at index 1 (diagonal element is a structural 0)";
    }
    CHECK(thrown);
    CHECK((x == Array1{2., 3., -1.}));
    printf("OK %d checks\n", g_checks);
    return 0;
}
