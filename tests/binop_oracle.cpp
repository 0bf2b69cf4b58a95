// binop_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU restatement of sprs's sparse binops that
// the device results are compared with bit for bit (tests/binop_oracle.py loads it).
//
//   oracle_binop_SUF    csmat_binop_same_storage_raw (sprs/src/sparse/binop.rs:229-271) with
//                       f = a + b, a - b or a * b (binop.rs:20-130), line by line: each outer
//                       dimension's two sorted index lists merged by nnz_or_zip, Left(a) ->
//                       f(a, 0), Right(b) -> f(0, b), Both(a, b) -> f(a, b), an entry kept when
//                       `!is_zero()` (v != 0.0: +-0.0 dropped, NaN kept).
//   oracle_scale_SUF    CsMatBase::map(|x| x * s) (binop.rs:132-163, csmat.rs:1289-1305): the
//                       structure is unchanged, nothing is dropped.
//
// SUF = index / indptr byte widths 44, 88, 48 (u32/u32, u64/u64, u32 indices + u64 indptr), as
// in oracle/sprs_oracle.cpp.  Single-threaded, like the reference.  -ffp-contract=off.
#include <cstddef>
#include <cstdint>

namespace {

enum { ADD = 0, SUB = 1, MUL = 2 };

inline double binop(int op, double a, double b) {
    return op == ADD ? a + b : op == SUB ? a - b : a * b;
}

// out arrays hold at least nnz(lhs) + nnz(rhs) entries; returns nnz of the result
template <typename I, typename Iptr>
size_t binop_raw(int op, size_t outer, const Iptr* lip, const I* lind, const double* ldat,
                 const Iptr* rip, const I* rind, const double* rdat, Iptr* out_indptr,
                 I* out_indices, double* out_data) {
    size_t nnz = 0;
    out_indptr[0] = 0;
    for (size_t dim = 0; dim < outer; ++dim) {
        // lv / rv: the outer dimension's views (indptr of a view may not start at 0)
        size_t l = (size_t)(lip[dim] - lip[0]), le = (size_t)(lip[dim + 1] - lip[0]);
        size_t r = (size_t)(rip[dim] - rip[0]), re = (size_t)(rip[dim + 1] - rip[0]);
        // nnz_or_zip: Left / Right / Both in ascending index order
        while (l < le || r < re) {
            size_t ind;
            double val;
            if (r == re || (l < le && lind[l] < rind[r])) {
                ind = (size_t)lind[l];
                val = binop(op, ldat[l], 0.0);
                ++l;
            } else if (l == le || rind[r] < lind[l]) {
                ind = (size_t)rind[r];
                val = binop(op, 0.0, rdat[r]);
                ++r;
            } else {
                ind = (size_t)lind[l];
                val = binop(op, ldat[l], rdat[r]);
                ++l;
                ++r;
            }
            if (val != 0.0) {
                out_indices[nnz] = (I)ind;
                out_data[nnz] = val;
                ++nnz;
            }
        }
        out_indptr[dim + 1] = (Iptr)nnz;
    }
    return nnz;
}

}  // namespace

#define ORACLE_BINOP(SUF, I, IPTR)                                                               \
    extern "C" size_t oracle_binop_##SUF(int op, size_t outer, const IPTR* lip, const I* lind,  \
                                         const double* ldat, const IPTR* rip, const I* rind,    \
                                         const double* rdat, IPTR* oip, I* oind, double* odat) { \
        return binop_raw<I, IPTR>(op, outer, lip, lind, ldat, rip, rind, rdat, oip, oind, odat); \
    }
ORACLE_BINOP(44, uint32_t, uint32_t)
ORACLE_BINOP(88, uint64_t, uint64_t)
ORACLE_BINOP(48, uint32_t, uint64_t)

extern "C" void oracle_scale(size_t nnz, const double* data, double s, double* out) {
    for (size_t k = 0; k < nnz; ++k) out[k] = data[k] * s;
}
