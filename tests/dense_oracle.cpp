// CPU oracle of the dense boundary (TEST INFRASTRUCTURE ONLY): to_dense.rs:12-30 assign_to_dense,
// csmat.rs:502-539 csr_from_dense and binop.rs:384-433 csmat_binop_dense_raw with the closures of
// add_dense_mat_same_ordering and mul_dense_mat_same_ordering, restated loop by loop.  Dense
// operands are (pointer, signed element strides rs, cs).  Built with -ffp-contract=off: every
// closure is its separately rounded IEEE operations, like the reference.
#include <cmath>
#include <cstddef>
#include <cstdint>

namespace {
inline double& el(double* p, int64_t rs, int64_t cs, uint64_t r, uint64_t c) {
    return p[(int64_t)r * rs + (int64_t)c * cs];
}
}  // namespace

extern "C" {

// assign_to_dense: for (sprow, drow) in outer_iterator().zip(axis_iter_mut(outer_axis)):
// drow[ind] = val.  storage 0 = CSR (outer = rows), 1 = CSC (outer = cols).
void oracle_assign_to_dense(int storage, uint64_t outer, const uint64_t* ip, const uint64_t* idx,
                            const double* data, double* out, int64_t rs, int64_t cs) {
    for (uint64_t o = 0; o < outer; ++o)
        for (uint64_t k = ip[o]; k < ip[o + 1]; ++k) {
            if (storage == 0)
                el(out, rs, cs, o, idx[k]) = data[k];
            else
                el(out, rs, cs, idx[k], o) = data[k];
        }
}

// csr_from_dense: epsilon clamped to zero unless > 0; the count loop builds indptr, the second
// loop pushes (col, x) for |x| > epsilon in row order.  Returns nnz; ip has rows + 1 entries,
// idx / data room for rows * cols.
uint64_t oracle_csr_from_dense(uint64_t rows, uint64_t cols, const double* m, int64_t rs,
                               int64_t cs, double epsilon, uint64_t* ip, uint64_t* idx,
                               double* data) {
    const double eps = epsilon > 0.0 ? epsilon : 0.0;
    uint64_t nnz = 0;
    ip[0] = 0;
    for (uint64_t r = 0; r < rows; ++r) {
        for (uint64_t c = 0; c < cols; ++c)
            if (std::fabs(el((double*)m, rs, cs, r, c)) > eps) ++nnz;
        ip[r + 1] = nnz;
    }
    uint64_t k = 0;
    for (uint64_t r = 0; r < rows; ++r)
        for (uint64_t c = 0; c < cols; ++c) {
            const double x = el((double*)m, rs, cs, r, c);
            if (std::fabs(x) > eps) {
                idx[k] = c;
                data[k] = x;
                ++k;
            }
        }
    return nnz;
}

// csmat_binop_dense_raw after its checks: out and rhs walked along the slowest axis (rows for
// CSR, columns for CSC), each dense lane enumerated and merged with the sparse vector
// (nnz_or_zip): Left (dense only) -> f(0, d), Both -> f(a, d).  op 0: (alpha*x) + (beta*y);
// op 2: (alpha*x)*y.
void oracle_binop_dense(int storage, uint64_t rows, uint64_t cols, const uint64_t* ip,
                        const uint64_t* idx, const double* data, int op, double alpha, double beta,
                        const double* rhs, int64_t rrs, int64_t rcs, double* out, int64_t ors,
                        int64_t ocs) {
    const uint64_t outer = storage == 0 ? rows : cols, inner = storage == 0 ? cols : rows;
    for (uint64_t o = 0; o < outer; ++o) {
        uint64_t k = ip[o];
        for (uint64_t i = 0; i < inner; ++i) {
            const uint64_t r = storage == 0 ? o : i, c = storage == 0 ? i : o;
            const double y = el((double*)rhs, rrs, rcs, r, c);
            double x = 0.0;
            if (k < ip[o + 1] && idx[k] == i) x = data[k++];
            double v;
            if (op == 0) {
                const double ax = alpha * x;
                const double by = beta * y;
                v = ax + by;
            } else {
                const double ax = alpha * x;
                v = ax * y;
            }
            el(out, ors, ocs, r, c) = v;
        }
    }
}

}  // extern "C"
