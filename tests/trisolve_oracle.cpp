// trisolve_oracle.cpp -- TEST INFRASTRUCTURE ONLY: a line-by-line restatement of the four
// dense-rhs solves of sprs::linalg::trisolve (sprs/src/sparse/linalg/trisolve.rs:30-262),
// early returns included, that the device solves (csrc/trisolve.cu) are compared with bit for
// bit.  Built with -ffp-contract=off (no FMA, like sprs) by tests/trisolve_oracle.py.
//
// Arrays: indptr u64 (zero-based), indices u32 ascending per outer dimension, f64 data.
// Each solve returns 0 for Ok, else 1 + the reason code and the failing index in *index:
//   0 "diagonal element is 0", 1 "... is a numeric 0", 2 "... is a structural 0"
// (the SPRS_B200_SINGULAR_* codes of include/sprs_b200.h).
#include <cstddef>
#include <cstdint>

namespace {

// CsVecView::get (the index's value, if stored): a binary search of the sorted indices
const double* get(const uint32_t* idx, const double* val, uint64_t s, uint64_t e, uint64_t i) {
    uint64_t lo = s, hi = e;
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (idx[mid] < i)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < e && idx[lo] == i ? val + lo : nullptr;
}

// lspsolve_csc_process_col (trisolve.rs:114-149)
int process_col(const uint64_t* ip, const uint32_t* idx, const double* val, uint64_t col,
                double* rhs) {
    const double* diag = get(idx, val, ip[col], ip[col + 1], col);
    if (!diag) return 1 + 2;
    if (*diag == 0.0) return 1 + 1;
    const double x = rhs[col] / *diag;
    rhs[col] = x;
    for (uint64_t k = ip[col]; k < ip[col + 1]; ++k) {
        if (idx[k] <= col) continue;
        rhs[idx[k]] -= val[k] * x;
    }
    return 0;
}

}  // namespace

extern "C" {

// trisolve.rs:30-73
int oracle_lsolve_csr(uint64_t n, const uint64_t* ip, const uint32_t* idx, const double* val,
                      double* rhs, uint64_t* index) {
    for (uint64_t row = 0; row < n; ++row) {
        double diag = 0.0;
        double x = rhs[row];
        for (uint64_t k = ip[row]; k < ip[row + 1]; ++k) {
            const uint64_t col = idx[k];
            if (col == row) {
                diag = val[k];
                continue;
            }
            if (col > row) continue;
            x -= val[k] * rhs[col];
        }
        if (diag == 0.0) {
            *index = row;
            return 1 + 0;
        }
        rhs[row] = x / diag;
    }
    return 0;
}

// trisolve.rs:219-262
int oracle_usolve_csr(uint64_t n, const uint64_t* ip, const uint32_t* idx, const double* val,
                      double* rhs, uint64_t* index) {
    for (uint64_t row = n; row-- > 0;) {
        double diag = 0.0;
        double x = rhs[row];
        for (uint64_t k = ip[row]; k < ip[row + 1]; ++k) {
            const uint64_t col = idx[k];
            if (col == row) {
                diag = val[k];
                continue;
            }
            if (col < row) continue;
            x -= val[k] * rhs[col];
        }
        if (diag == 0.0) {
            *index = row;
            return 1 + 1;
        }
        rhs[row] = x / diag;
    }
    return 0;
}

// trisolve.rs:85-112
int oracle_lsolve_csc(uint64_t n, const uint64_t* ip, const uint32_t* idx, const double* val,
                      double* rhs, uint64_t* index) {
    for (uint64_t col = 0; col < n; ++col) {
        const int st = process_col(ip, idx, val, col, rhs);
        if (st) {
            *index = col;
            return st;
        }
    }
    return 0;
}

// trisolve.rs:161-210
int oracle_usolve_csc(uint64_t n, const uint64_t* ip, const uint32_t* idx, const double* val,
                      double* rhs, uint64_t* index) {
    for (uint64_t col = n; col-- > 0;) {
        const double* diag = get(idx, val, ip[col], ip[col + 1], col);
        if (!diag) {
            *index = col;
            return 1 + 2;
        }
        if (*diag == 0.0) {
            *index = col;
            return 1 + 1;
        }
        const double x = rhs[col] / *diag;
        rhs[col] = x;
        for (uint64_t k = ip[col]; k < ip[col + 1]; ++k) {
            if (idx[k] >= col) continue;
            rhs[idx[k]] -= val[k] * x;
        }
    }
    return 0;
}

// Depth of the dependency graph of a solve (for reports): level[i] = 1 + the largest level of
// the rows i depends on, over the triangle the solve uses.  csr: rows of (ip, idx) are rows of
// the matrix, else columns.  Returns the largest level (0 for n == 0).
uint64_t oracle_levels(uint64_t n, const uint64_t* ip, const uint32_t* idx, int upper, int csr,
                       uint32_t* level) {
    uint64_t depth = 0;
    for (uint64_t i = 0; i < n; ++i) level[i] = 1;
    for (uint64_t t = 0; t < n; ++t) {
        const uint64_t o = upper ? n - 1 - t : t;  // processing order
        for (uint64_t k = ip[o]; k < ip[o + 1]; ++k) {
            const uint64_t j = idx[k];
            // csr: row o depends on column j < o (lower); csc: row j > o depends on column o
            const bool dep = (upper != 0) == (csr != 0) ? j > o : j < o;
            if (!dep) continue;
            if (csr) {
                if (level[j] + 1 > level[o]) level[o] = level[j] + 1;
            } else if (level[o] + 1 > level[j]) {
                level[j] = level[o] + 1;
            }
        }
        if (level[o] > depth) depth = level[o];
    }
    return n ? depth : 0;
}

}  // extern "C"
