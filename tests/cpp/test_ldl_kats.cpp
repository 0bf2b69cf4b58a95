// test_ldl_kats.cpp -- the sprs-ldl crate's tests (sprs-ldl/src/lib.rs, `mod test`) replayed
// through the C++ host mirror (include/sprs_b200.hpp) on the GPU, with the panics, a singular
// update and the recovery after it.  Built and run by tests/test_gpu_ldl.py::test_cpp_ldl_kats
// (and on the emulator by tests/test_emu_ldl.py); exits non-zero on the first failure.
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

template <class F>
static bool panics_with(F f, const char* msg) {
    try {
        f();
    } catch (const Panic& p) {
        return std::string(p.what()) == msg;
    }
    return false;
}

static CsMat test_mat1() {
    return CsMat::new_csc({10, 10}, {0, 2, 5, 6, 7, 13, 14, 17, 20, 24, 28},
                          {0, 8, 1, 4, 9, 2, 3, 1, 4, 6, 7, 8, 9, 5, 4, 6, 9, 4, 7, 8, 0, 4, 7, 8,
                           1, 4, 6, 9},
                          {1.7, 0.13, 1., 0.02, 0.01, 1.5, 1.1, 0.02, 2.6, 0.16, 0.09, 0.52, 0.53,
                           1.2, 0.16, 1.3, 0.56, 0.09, 1.6, 0.11, 0.13, 0.52, 0.11, 1.4, 0.01,
                           0.53, 0.56, 3.1});
}

int main() {
    using ldl::LdlNumeric;
    using ldl::LdlSymbolic;
    using ldl::SymmetryCheck;
    // test_factor1 / test_factor_solve1: expected_factors1 and expected_res1
    const CsMat a = test_mat1();
    LdlNumeric f = LdlNumeric::new_(a);
    const CsMatI<size_t> l = f.l();
    CHECK((l.indptr() == std::vector<size_t>{0, 1, 3, 3, 3, 7, 7, 10, 12, 13, 13}));
    CHECK((l.indices() == std::vector<size_t>{8, 4, 9, 6, 7, 8, 9, 7, 8, 9, 8, 9, 9}));
    CHECK((l.data() == Array1{0.076470588235294124, 0.02, 0.01, 0.061547930450838589,
                              0.034620710878596701, 0.20003077396522542, 0.20380058470533929,
                              -0.0042935346524025902, -0.024807089102770519, 0.40878266366119237,
                              0.05752526570865537, -0.010068305077340346,
                              -0.071852278207562709}));
    CHECK((f.d() == Array1{1.7, 1., 1.5, 1.1000000000000001, 2.5996000000000001, 1.2,
                           1.290152331127866, 1.5968603527854308, 1.2799646117414738,
                           2.7695677698030283}));
    const Array1 b = {0.287, 0.22, 0.45, 0.44, 2.486, 0.72, 1.55, 1.424, 1.621, 3.759};
    const Array1 want = {0.099999999999999992, 0.19999999999999998, 0.29999999999999999,
                         0.39999999999999997, 0.5, 0.59999999999999998, 0.70000000000000007,
                         0.79999999999999993, 0.90000000000000002, 0.99999999999999989};
    CHECK(f.solve(b) == want);
    CHECK(f.nnz() == 13 && f.problem_size() == 10);
    // test_solve1's diag_solve step: expected_lsolve_res1 / expected_dsolve_res1
    Array1 x = {0.28699999999999998, 0.22, 0.45000000000000001, 0.44, 2.4816000000000003,
                0.71999999999999997, 1.3972626557931991, 1.3440844395148306, 1.0599997771886431,
                2.7695677698030279};
    linalg::diag_solve(f.d(), x);
    CHECK((x == Array1{0.16882352941176471, 0.22, 0.29999999999999999, 0.39999999999999997,
                       0.95460840129250657, 0.59999999999999998, 1.0830214557467768,
                       0.84170443406044937, 0.82814772179243734, 0.99999999999999989}));
    // permuted_ldl_solve
    const CsMat p = CsMat::new_csc({4, 4}, {0, 2, 4, 6, 8}, {0, 3, 1, 2, 1, 2, 0, 3},
                                   {1., 2., 21., 6., 6., 2., 2., 8.});
    LdlNumeric fp = LdlNumeric::new_perm(p, {0, 2, 1, 3}, SymmetryCheck::CheckSymmetry);
    CHECK((fp.solve({9., 60., 18., 34.}) == Array1{1., 2., 3., 4.}));
    // the panics, in the reference's order: square, symmetry, permutation
    const CsMat rect = CsMat::new_({2, 3}, {0, 1, 2}, {0, 1}, {1., 1.});
    CHECK(panics_with([&] { LdlNumeric::new_perm(rect, {0, 1}, SymmetryCheck::CheckSymmetry); },
                      "matrix should be square"));
    const CsMat nonsym = CsMat::new_({3, 3}, {0, 2, 3, 4}, {0, 1, 1, 2}, {1., 5., 1., 1.});
    CHECK(!ldl::is_symmetric(nonsym) && ldl::is_symmetric(a));
    CHECK(panics_with([&] { LdlNumeric::new_perm(nonsym, {0, 1, 1}, SymmetryCheck::CheckSymmetry); },
                      "Matrix is not symmetric"));
    CHECK(panics_with([&] { LdlNumeric::new_perm(nonsym, {0, 1, 1}, SymmetryCheck::DontCheckSymmetry); },
                      "assertion failed: perm_is_valid(&perm)"));
    // a singular update: D_1 = 1 - 1 * 1 == 0; l, d, solve throw until an update succeeds
    const CsMat good = CsMat::new_({3, 3}, {0, 2, 4, 5}, {0, 1, 0, 1, 2}, {1., 1., 1., 2., 4.});
    const CsMat bad = CsMat::new_({3, 3}, {0, 2, 4, 5}, {0, 1, 0, 1, 2}, {1., 1., 1., 1., 4.});
    LdlNumeric g = LdlNumeric::new_(good);
    const Array1 xg = g.solve({2., 3., 4.});
    CHECK((xg == Array1{1., 1., 1.}));
    bool thrown = false;
    try {
        g.update(bad);
    } catch (const linalg::SingularMatrix& e) {
        thrown = e.index == 1 && e.reason == "diagonal element is a numeric 0";
    }
    CHECK(thrown);
    int refused = 0;
    try { g.d(); } catch (const linalg::SingularMatrix&) { ++refused; }
    try { g.l(); } catch (const linalg::SingularMatrix&) { ++refused; }
    try { g.solve({2., 3., 4.}); } catch (const linalg::SingularMatrix&) { ++refused; }
    CHECK(refused == 3);
    g.update(good);
    CHECK(g.solve({2., 3., 4.}) == xg);
    // another pattern: refused before any work, the factor unchanged
    const CsMat other = CsMat::new_({3, 3}, {0, 1, 2, 3}, {0, 1, 2}, {1., 2., 4.});
    CHECK(panics_with([&] { g.update(other); },
                      "ldl update: the matrix's pattern differs from the symbolic factorization's"));
    CHECK(g.solve({2., 3., 4.}) == xg);
    printf("OK %d checks\n", g_checks);
    return 0;
}
