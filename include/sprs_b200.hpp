// sprs_b200.hpp -- C++ host mirror of the sprs operator API for the product path.
//
// The reference's host language is Rust; this image has no Rust toolchain (DESIGN.md),
// so the host side above the C ABI is written in C++ (the reference is compiled code)
// with the SAME names, argument meaning and error behaviour as sprs:
//
//   sprs::CsMatI<I, Iptr>, CsMat = CsMatI<size_t>     sprs/src/sparse.rs:94-129
//   CsMat::new_ / new_csc / eye / zero                 sprs/src/sparse/csmat.rs
//   &a * &b  (sparse, Array2, Array1, CsVec), dot()    csmat.rs:1866-2178, vec.rs:1084-1131
//   sprs::prod::mul_acc_mat_vec_csr / csr_mulacc_dense_{row,col}maj / ...   prod.rs
//   sprs::smmp::mul_csr_csr                            smmp.rs:196-237
//   &a + &b, &a - &b, &a * s, binop::mul_mat_same_storage   binop.rs:20-163
//   to_dense, assign_to_dense, csr/csc_from_dense, &a + &d,
//   binop::{add,mul}_dense_mat_same_ordering   to_dense.rs, csmat.rs:502-549, binop.rs:273-433
//
// Contract violations throw sprs::Panic carrying the reference's panic message
// ("Dimension mismatch", "Storage mismatch"; Guidelines.rst:9-27); device failures
// throw sprs::ThirdPartyError(code, msg) (LinalgError::ThirdPartyError, errors.rs:70).
// Host arrays are owned here (as Rust owns its Vecs); the device mirror is an opaque
// handle freed in the destructor (the UMFPACK `impl Drop` pattern).  Every product is
// a call into libsprs_b200.so -- there is no CPU implementation in this header.
// The Rust crates in rust/ are the same wrapper in the reference's own language.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <functional>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "sprs_b200.h"

namespace sprs {

struct Panic : std::logic_error {
    using std::logic_error::logic_error;
};
struct ThirdPartyError : std::runtime_error {
    int code;
    ThirdPartyError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

enum class CompressedStorage { CSR, CSC };
constexpr CompressedStorage CSR = CompressedStorage::CSR;
constexpr CompressedStorage CSC = CompressedStorage::CSC;

// One context per thread, like the reference's thread-local ThreadingStrategy (smmp.rs:35-38)
class Context {
   public:
    explicit Context(int device = 0) {
        const int st = sprs_b200_ctx_create(device, &h_);
        if (st != SPRS_B200_OK) throw ThirdPartyError(st, sprs_b200_last_error(nullptr));
    }
    ~Context() { sprs_b200_ctx_destroy(h_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    sprs_b200_ctx* handle() const { return h_; }
    void check(int st) const {
        if (st == SPRS_B200_OK) return;
        if (st == SPRS_B200_ERR_DIMENSION) throw Panic("Dimension mismatch");
        if (st == SPRS_B200_ERR_STORAGE) throw Panic("Storage mismatch");
        if (st == SPRS_B200_ERR_INDEX_RANGE) throw Panic(sprs_b200_last_error(h_));
        throw ThirdPartyError(st, sprs_b200_last_error(h_));
    }
    static Context& thread_default() {
        static thread_local Context ctx(0);
        return ctx;
    }

   private:
    sprs_b200_ctx* h_ = nullptr;
};

// ndarray stand-ins: Array1 = std::vector<double>; Array2 keeps element strides so that
// C-order, F-order and transposed views are all expressible (ArrayView semantics).
using Array1 = std::vector<double>;
struct Array2 {
    size_t rows = 0, cols = 0;
    std::ptrdiff_t rs = 0, cs = 0;  // element strides
    std::vector<double> data;
    static Array2 zeros(size_t r, size_t c) {  // Array::zeros((r, c))  -> C order
        Array2 a;
        a.rows = r; a.cols = c; a.rs = (std::ptrdiff_t)c; a.cs = 1;
        a.data.assign(r * c, 0.0);
        return a;
    }
    static Array2 zeros_f(size_t r, size_t c) {  // Array::zeros((r, c).f()) -> F order
        Array2 a;
        a.rows = r; a.cols = c; a.rs = 1; a.cs = (std::ptrdiff_t)r;
        a.data.assign(r * c, 0.0);
        return a;
    }
    static Array2 from_rows(const std::vector<std::vector<double>>& v) {  // arr2(&[[..],..])
        Array2 a = zeros(v.size(), v.empty() ? 0 : v[0].size());
        for (size_t i = 0; i < a.rows; ++i)
            for (size_t j = 0; j < a.cols; ++j) a(i, j) = v[i][j];
        return a;
    }
    Array2 reversed_axes() const {  // zero-copy in ndarray; a copy of the header here
        Array2 t = *this;
        std::swap(t.rows, t.cols);
        std::swap(t.rs, t.cs);
        return t;
    }
    Array2 to_f_order() const {
        Array2 f = zeros_f(rows, cols);
        for (size_t i = 0; i < rows; ++i)
            for (size_t j = 0; j < cols; ++j) f(i, j) = (*this)(i, j);
        return f;
    }
    bool is_standard_layout() const { return cs == 1 && rs == (std::ptrdiff_t)cols; }
    double& operator()(size_t i, size_t j) { return data[i * rs + j * cs]; }
    double operator()(size_t i, size_t j) const { return data[i * rs + j * cs]; }
    bool operator==(const Array2& o) const {
        if (rows != o.rows || cols != o.cols) return false;
        for (size_t i = 0; i < rows; ++i)
            for (size_t j = 0; j < cols; ++j)
                if ((*this)(i, j) != o(i, j)) return false;
        return true;
    }
};

template <class I = size_t>
struct CsVecI {  // CsVecBase (sparse.rs:166-182)
    size_t dim = 0;
    std::vector<I> indices;
    std::vector<double> data;
    CsVecI() = default;
    CsVecI(size_t d, std::vector<I> i, std::vector<double> v)
        : dim(d), indices(std::move(i)), data(std::move(v)) {
        if (indices.size() != data.size()) throw Panic("indices and data lengths differ");
        for (size_t k = 0; k < indices.size(); ++k)
            if ((size_t)indices[k] >= dim || (k && indices[k - 1] >= indices[k]))
                throw Panic("Unsorted or out-of-bounds indices");
    }
    static CsVecI empty(size_t d) { return CsVecI(d, {}, {}); }
    size_t nnz() const { return indices.size(); }
    bool operator==(const CsVecI& o) const {
        return dim == o.dim && indices == o.indices && data == o.data;
    }
};
using CsVec = CsVecI<size_t>;

template <class I = size_t, class Iptr = I>
class CsMatI {
    static_assert(sizeof(I) == 4 || sizeof(I) == 8, "index types are 4 or 8 bytes");
    static_assert(sizeof(Iptr) == 4 || sizeof(Iptr) == 8, "indptr types are 4 or 8 bytes");

   public:
    CsMatI(CompressedStorage st, std::pair<size_t, size_t> shape, std::vector<Iptr> indptr,
           std::vector<I> indices, std::vector<double> data)
        : storage_(st), rows_(shape.first), cols_(shape.second), indptr_(std::move(indptr)),
          indices_(std::move(indices)), data_(std::move(data)) {
        check_structure();
    }
    // CsMat::new / new_csc (csmat.rs); `new_` because `new` is a C++ keyword
    static CsMatI new_(std::pair<size_t, size_t> shape, std::vector<Iptr> ip, std::vector<I> ind,
                       std::vector<double> d) {
        return CsMatI(CSR, shape, std::move(ip), std::move(ind), std::move(d));
    }
    static CsMatI new_csc(std::pair<size_t, size_t> shape, std::vector<Iptr> ip,
                          std::vector<I> ind, std::vector<double> d) {
        return CsMatI(CSC, shape, std::move(ip), std::move(ind), std::move(d));
    }
    static CsMatI eye(size_t n) {
        std::vector<Iptr> ip(n + 1);
        std::vector<I> ind(n);
        for (size_t i = 0; i <= n; ++i) ip[i] = (Iptr)i;
        for (size_t i = 0; i < n; ++i) ind[i] = (I)i;
        return CsMatI(CSR, {n, n}, ip, ind, std::vector<double>(n, 1.0));
    }
    static CsMatI zero(std::pair<size_t, size_t> shape) {
        return CsMatI(CSR, shape, std::vector<Iptr>(shape.first + 1, 0), {}, {});
    }
    CsMatI(const CsMatI& o)
        : storage_(o.storage_), rows_(o.rows_), cols_(o.cols_), indptr_(o.indptr_),
          indices_(o.indices_), data_(o.data_) {}
    CsMatI(CsMatI&& o) noexcept { *this = std::move(o); }
    CsMatI& operator=(CsMatI&& o) noexcept {
        release();
        storage_ = o.storage_; rows_ = o.rows_; cols_ = o.cols_;
        indptr_ = std::move(o.indptr_); indices_ = std::move(o.indices_); data_ = std::move(o.data_);
        dev_ = o.dev_; o.dev_ = nullptr;
        return *this;
    }
    ~CsMatI() { release(); }

    size_t rows() const { return rows_; }
    size_t cols() const { return cols_; }
    size_t nnz() const { return indptr_.empty() ? 0 : (size_t)(indptr_.back() - indptr_.front()); }
    bool is_csr() const { return storage_ == CSR; }
    bool is_csc() const { return storage_ == CSC; }
    CompressedStorage storage() const { return storage_; }
    size_t outer_dims() const { return is_csr() ? rows_ : cols_; }
    size_t inner_dims() const { return is_csr() ? cols_ : rows_; }
    const std::vector<Iptr>& indptr() const { return indptr_; }
    const std::vector<I>& indices() const { return indices_; }
    const std::vector<double>& data() const { return data_; }
    bool operator==(const CsMatI& o) const {  // derive(PartialEq) on CsMatBase
        return storage_ == o.storage_ && rows_ == o.rows_ && cols_ == o.cols_ &&
               indptr_ == o.indptr_ && indices_ == o.indices_ && data_ == o.data_;
    }

    // transpose_view / transpose_into: same arrays, other storage, swapped shape
    CsMatI transpose_into() const {
        return CsMatI(is_csr() ? CSC : CSR, {cols_, rows_}, indptr_, indices_, data_);
    }
    CsMatI transpose_view() const { return transpose_into(); }
    // slice_outer (slicing.rs:65-89); the result keeps a NON-zero-based indptr
    // (indptr.rs:122-124) which the upload rebases like proper_indptr().
    CsMatI slice_outer(size_t start, size_t stop) const {
        std::vector<Iptr> ip(indptr_.begin() + start, indptr_.begin() + stop + 1);
        const size_t s = (size_t)(indptr_[start] - indptr_[0]), e = (size_t)(indptr_[stop] - indptr_[0]);
        std::vector<I> ind(indices_.begin() + s, indices_.begin() + e);
        std::vector<double> d(data_.begin() + s, data_.begin() + e);
        const size_t n = stop - start;
        return CsMatI(storage_, is_csr() ? std::make_pair(n, cols_) : std::make_pair(rows_, n),
                      std::move(ip), std::move(ind), std::move(d));
    }
    // to_other_storage (csmat.rs:1405-1426) through the device counting sort
    CsMatI to_other_storage() const {
        // raw::convert_mat_storage asserts that rows() fits the index type before any work
        // (csmat.rs:1794-1797; sprs/tests/gh374.rs)
        if ((uint64_t)rows_ > (uint64_t)std::numeric_limits<I>::max())
            throw Panic("Index type is not large enough to hold the number of rows requested");
        Context& ctx = Context::thread_default();
        sprs_b200_csmat* t = nullptr;
        ctx.check(sprs_b200_csmat_to_other_storage(ctx.handle(), device(), &t));
        CsMatI out = download(ctx, t, is_csr() ? CSC : CSR, rows_, cols_);
        sprs_b200_csmat_free(t);
        return out;
    }
    CsMatI to_csr() const { return is_csr() ? *this : to_other_storage(); }
    CsMatI to_csc() const { return is_csc() ? *this : to_other_storage(); }

    // device mirror (lazy upload)
    const sprs_b200_csmat* device() const {
        if (!dev_) {
            Context& ctx = Context::thread_default();
            ctx.check(sprs_b200_csmat_upload(ctx.handle(), is_csr() ? SPRS_B200_CSR : SPRS_B200_CSC,
                                             rows_, cols_, indptr_.data(), (int)sizeof(Iptr),
                                             indices_.data(), (int)sizeof(I), data_.data(), &dev_));
        }
        return dev_;
    }
    static CsMatI download(Context& ctx, const sprs_b200_csmat* m, CompressedStorage st,
                           size_t rows, size_t cols) {
        const size_t outer = st == CSR ? rows : cols;
        std::vector<Iptr> ip(outer + 1);
        std::vector<I> ind(sprs_b200_csmat_nnz(m));
        std::vector<double> d(ind.size());
        ctx.check(sprs_b200_csmat_download(ctx.handle(), m, ip.data(), (int)sizeof(Iptr),
                                           ind.data(), (int)sizeof(I), d.data()));
        return CsMatI(st, {rows, cols}, std::move(ip), std::move(ind), std::move(d), 0);
    }

    // to_dense (csmat.rs:1127-1134) on the device: C order, stored values as bits, +0.0 elsewhere
    Array2 to_dense() const {
        Array2 out = Array2::zeros(rows_, cols_);
        if (rows_ && cols_) {
            Context& ctx = Context::thread_default();
            ctx.check(sprs_b200_csmat_to_dense(ctx.handle(), device(), out.data.data(), cols_));
        }
        return out;
    }
    // csr_from_dense / csc_from_dense (csmat.rs:502-549) on the device: |x| > epsilon kept
    // (epsilon clamped to +0.0 unless > 0), values copied as bits
    static CsMatI csr_from_dense(const Array2& m, double epsilon) { return from_dense(m, epsilon, CSR); }
    static CsMatI csc_from_dense(const Array2& m, double epsilon) { return from_dense(m, epsilon, CSC); }

    double to_dense_at(size_t r, size_t c) const {
        const size_t o = is_csr() ? r : c, in = is_csr() ? c : r;
        for (size_t k = (size_t)(indptr_[o] - indptr_[0]); k < (size_t)(indptr_[o + 1] - indptr_[0]); ++k)
            if ((size_t)indices_[k] == in) return data_[k];
        return 0.0;
    }

    // `.dot()` forms (csmat.rs:2101-2178) are the operators
    template <class R>
    auto dot(const R& rhs) const { return *this * rhs; }

   private:
    static CsMatI from_dense(const Array2& m, double epsilon, CompressedStorage st) {
        Context& ctx = Context::thread_default();
        sprs_b200_csmat* t = nullptr;
        const bool empty = m.rows == 0 || m.cols == 0;
        ctx.check(sprs_b200_csmat_from_dense(ctx.handle(), st == CSR ? SPRS_B200_CSR : SPRS_B200_CSC,
                                             m.rows, m.cols, empty ? nullptr : m.data.data(),
                                             empty ? 0 : m.rs, empty ? 0 : m.cs, epsilon, &t));
        CsMatI out = download(ctx, t, st, m.rows, m.cols);
        sprs_b200_csmat_free(t);
        return out;
    }
    CsMatI(CompressedStorage st, std::pair<size_t, size_t> shape, std::vector<Iptr> ip,
           std::vector<I> ind, std::vector<double> d, int /*trusted*/)
        : storage_(st), rows_(shape.first), cols_(shape.second), indptr_(std::move(ip)),
          indices_(std::move(ind)), data_(std::move(d)) {}
    void release() {
        if (dev_) sprs_b200_csmat_free(dev_);
        dev_ = nullptr;
    }
    void check_structure() const {  // check_compressed_structure (sparse.rs:300-369)
        if (indptr_.size() != outer_dims() + 1) throw Panic("Indptr length does not match dimension");
        for (size_t o = 0; o < outer_dims(); ++o) {
            if (indptr_[o + 1] < indptr_[o]) throw Panic("Unsorted indptr");
            for (size_t k = (size_t)(indptr_[o] - indptr_[0]); k < (size_t)(indptr_[o + 1] - indptr_[0]); ++k) {
                if (k >= indices_.size() || k >= data_.size()) throw Panic("Indices or data shorter than nnz");
                if ((size_t)indices_[k] >= inner_dims()) throw Panic("Out of bounds index");
                if (k > (size_t)(indptr_[o] - indptr_[0]) && indices_[k - 1] >= indices_[k])
                    throw Panic("Unsorted indices");
            }
        }
    }
    CompressedStorage storage_ = CSR;
    size_t rows_ = 0, cols_ = 0;
    std::vector<Iptr> indptr_;
    std::vector<I> indices_;
    std::vector<double> data_;
    mutable sprs_b200_csmat* dev_ = nullptr;
};
using CsMat = CsMatI<size_t, size_t>;

// ------------------------------------------------------------------------------------
namespace smmp {
// smmp::mul_csr_csr (smmp.rs:196-237).  The output Vecs are allocated by the CALLER
// between the symbolic and numeric calls, as in the reference.
template <class I, class Iptr>
CsMatI<I, Iptr> mul_csr_csr(const CsMatI<I, Iptr>& lhs, const CsMatI<I, Iptr>& rhs) {
    if (lhs.cols() != rhs.rows()) throw Panic("Dimension mismatch");  // assert_eq! smmp.rs:207
    if (!lhs.is_csr() || !rhs.is_csr()) throw Panic("Storage mismatch");
    Context& ctx = Context::thread_default();
    sprs_b200_spgemm* plan = nullptr;
    uint64_t nnz_c = 0;
    ctx.check(sprs_b200_spgemm_symbolic(ctx.handle(), lhs.device(), rhs.device(), &plan, &nnz_c));
    std::vector<Iptr> ip(lhs.rows() + 1);
    std::vector<I> ind(nnz_c);
    std::vector<double> d(nnz_c);
    const int st = sprs_b200_spgemm_numeric(ctx.handle(), plan, ip.data(), (int)sizeof(Iptr),
                                            ind.data(), (int)sizeof(I), d.data());
    sprs_b200_spgemm_free(plan);
    ctx.check(st);
    return CsMatI<I, Iptr>::new_({lhs.rows(), rhs.cols()}, std::move(ip), std::move(ind),
                                 std::move(d));
}
}  // namespace smmp

namespace prod {
// prod::mul_acc_mat_vec_csr (prod.rs:103-127): res_vec += mat * in_vec
template <class I, class Iptr>
void mul_acc_mat_vec_csr(const CsMatI<I, Iptr>& mat, const Array1& in_vec, Array1& res_vec) {
    if (mat.cols() != in_vec.size() || mat.rows() != res_vec.size()) throw Panic("Dimension mismatch");
    if (!mat.is_csr()) throw Panic("Storage mismatch");
    Context& ctx = Context::thread_default();
    ctx.check(sprs_b200_mul_acc_mat_vec_csr(ctx.handle(), mat.device(), in_vec.data(),
                                            in_vec.size(), res_vec.data(), res_vec.size()));
}
// prod::mul_acc_mat_vec_csc (prod.rs:74-99)
template <class I, class Iptr>
void mul_acc_mat_vec_csc(const CsMatI<I, Iptr>& mat, const Array1& in_vec, Array1& res_vec) {
    if (mat.cols() != in_vec.size() || mat.rows() != res_vec.size()) throw Panic("Dimension mismatch");
    if (!mat.is_csc()) throw Panic("Storage mismatch");
    Context& ctx = Context::thread_default();
    ctx.check(sprs_b200_mul_acc_mat_vec_csc(ctx.handle(), mat.device(), in_vec.data(),
                                            in_vec.size(), res_vec.data(), res_vec.size()));
}
#define SPRS_DENSE_FN(NAME, WANT_CSR)                                                          \
    template <class I, class Iptr>                                                             \
    void NAME(const CsMatI<I, Iptr>& lhs, const Array2& rhs, Array2& out) {                    \
        if (lhs.cols() != rhs.rows || lhs.rows() != out.rows || rhs.cols != out.cols)          \
            throw Panic("Dimension mismatch");                                                 \
        if (lhs.is_csr() != WANT_CSR) throw Panic("Storage mismatch");                         \
        Context& ctx = Context::thread_default();                                              \
        ctx.check(sprs_b200_##NAME(ctx.handle(), lhs.device(), rhs.data.data(), rhs.rows,      \
                                   rhs.cols, rhs.rs, rhs.cs, out.data.data(), out.rows,        \
                                   out.cols, out.rs, out.cs));                                 \
    }
SPRS_DENSE_FN(csr_mulacc_dense_rowmaj, true)   // prod.rs:189-214
SPRS_DENSE_FN(csr_mulacc_dense_colmaj, true)   // prod.rs:274-298
SPRS_DENSE_FN(csc_mulacc_dense_rowmaj, false)  // prod.rs:219-241
SPRS_DENSE_FN(csc_mulacc_dense_colmaj, false)  // prod.rs:246-269
#undef SPRS_DENSE_FN
}  // namespace prod

// ---- operators: the `impl Mul` blocks -------------------------------------------------
// csmat_mul_csmat (csmat.rs:1895-1949)
template <class I, class Iptr>
CsMatI<I, Iptr> operator*(const CsMatI<I, Iptr>& lhs, const CsMatI<I, Iptr>& rhs) {
    if (lhs.is_csr() && rhs.is_csr()) return smmp::mul_csr_csr(lhs, rhs);
    if (lhs.is_csr() && rhs.is_csc()) return smmp::mul_csr_csr(lhs, rhs.to_other_storage());
    if (lhs.is_csc() && rhs.is_csr()) {
        const auto rhs_csc = rhs.to_other_storage();
        return smmp::mul_csr_csr(rhs_csc.transpose_view(), lhs.transpose_view()).transpose_into();
    }
    return smmp::mul_csr_csr(rhs.transpose_view(), lhs.transpose_view()).transpose_into();
}

// ---- the `impl Add / Sub / Mul<N>` blocks and binop::mul_mat_same_storage (binop.rs:20-163)
namespace binop {
namespace detail {
// csmat_binop (binop.rs:178-271) on the device: the result in lhs's storage, entries whose
// result is 0.0 dropped; `rhs_dev` has lhs's storage
template <class I, class Iptr>
CsMatI<I, Iptr> csmat_binop(const CsMatI<I, Iptr>& lhs, const sprs_b200_csmat* rhs_dev, int op) {
    Context& ctx = Context::thread_default();
    sprs_b200_csmat* c = nullptr;
    ctx.check(sprs_b200_csmat_binop(ctx.handle(), lhs.device(), rhs_dev, op, &c));
    CsMatI<I, Iptr> out = CsMatI<I, Iptr>::download(ctx, c, lhs.storage(), lhs.rows(), lhs.cols());
    sprs_b200_csmat_free(c);
    return out;
}
// Add / Sub: the shapes are asserted first, then rhs is converted to lhs's storage
template <class I, class Iptr>
CsMatI<I, Iptr> add_or_sub(const CsMatI<I, Iptr>& lhs, const CsMatI<I, Iptr>& rhs, int op) {
    if (lhs.rows() != rhs.rows() || lhs.cols() != rhs.cols()) throw Panic("Dimension mismatch");
    if (lhs.storage() == rhs.storage()) return csmat_binop(lhs, rhs.device(), op);
    Context& ctx = Context::thread_default();
    sprs_b200_csmat* t = nullptr;
    ctx.check(sprs_b200_csmat_to_other_storage(ctx.handle(), rhs.device(), &t));
    sprs_b200_csmat* c = nullptr;
    const int st = sprs_b200_csmat_binop(ctx.handle(), lhs.device(), t, op, &c);
    sprs_b200_csmat_free(t);
    ctx.check(st);
    CsMatI<I, Iptr> out = CsMatI<I, Iptr>::download(ctx, c, lhs.storage(), lhs.rows(), lhs.cols());
    sprs_b200_csmat_free(c);
    return out;
}
}  // namespace detail

// binop::mul_mat_same_storage (binop.rs:115-130): element-wise product; mixed storage panics
template <class I, class Iptr>
CsMatI<I, Iptr> mul_mat_same_storage(const CsMatI<I, Iptr>& lhs, const CsMatI<I, Iptr>& rhs) {
    if (lhs.rows() != rhs.rows() || lhs.cols() != rhs.cols()) throw Panic("Dimension mismatch");
    if (lhs.storage() != rhs.storage()) throw Panic("Storage mismatch");
    return detail::csmat_binop(lhs, rhs.device(), SPRS_B200_BINOP_MUL);
}
}  // namespace binop

// `&A + &B` (binop.rs:20-65)
template <class I, class Iptr>
CsMatI<I, Iptr> operator+(const CsMatI<I, Iptr>& lhs, const CsMatI<I, Iptr>& rhs) {
    return binop::detail::add_or_sub(lhs, rhs, SPRS_B200_BINOP_ADD);
}
// `&A - &B` (binop.rs:67-112)
template <class I, class Iptr>
CsMatI<I, Iptr> operator-(const CsMatI<I, Iptr>& lhs, const CsMatI<I, Iptr>& rhs) {
    return binop::detail::add_or_sub(lhs, rhs, SPRS_B200_BINOP_SUB);
}
// `&A * s` (binop.rs:132-163 -> CsMatBase::map): same structure, every value times s
template <class I, class Iptr>
CsMatI<I, Iptr> operator*(const CsMatI<I, Iptr>& a, double s) {
    Context& ctx = Context::thread_default();
    sprs_b200_csmat* c = nullptr;
    ctx.check(sprs_b200_csmat_scale(ctx.handle(), a.device(), s, &c));
    CsMatI<I, Iptr> out = CsMatI<I, Iptr>::download(ctx, c, a.storage(), a.rows(), a.cols());
    sprs_b200_csmat_free(c);
    return out;
}
// ---- the dense boundary: to_dense.rs, binop.rs:273-433, csmat.rs:1951-1987
namespace detail {
// element strides as ndarray has them: an array with a zero-length axis has all-zero strides
inline std::pair<std::ptrdiff_t, std::ptrdiff_t> nd_strides(const Array2& a) {
    if (a.rows == 0 || a.cols == 0) return {0, 0};
    return {a.rs, a.cs};
}
// utils::fastest_axis (sparse.rs:400-406): Axis(0) iff strides[1] > strides[0]
inline int fastest_axis(const Array2& a) {
    const auto st = nd_strides(a);
    return st.second > st.first ? 0 : 1;
}
inline void binop_dense(const sprs_b200_csmat* lhs, int op, double alpha, double beta,
                        const Array2& rhs, Array2& out) {
    Context& ctx = Context::thread_default();
    const auto r = nd_strides(rhs), o = nd_strides(out);
    ctx.check(sprs_b200_csmat_binop_dense(ctx.handle(), lhs, op, alpha, beta, rhs.data.data(),
                                          rhs.rows, rhs.cols, r.first, r.second, out.data.data(),
                                          out.rows, out.cols, o.first, o.second));
}
}  // namespace detail

// assign_to_dense (to_dense.rs:12-30): stored values into array as bits, the rest untouched
template <class I, class Iptr>
void assign_to_dense(Array2& array, const CsMatI<I, Iptr>& m) {
    if (m.cols() != array.cols || m.rows() != array.rows) throw Panic("Dimension mismatch");
    Context& ctx = Context::thread_default();
    const auto st = detail::nd_strides(array);
    ctx.check(sprs_b200_assign_to_dense(ctx.handle(), m.device(), array.data.data(), array.rows,
                                        array.cols, st.first, st.second));
}

namespace binop {
// add_dense_mat_same_ordering (binop.rs:279-323): (alpha*x) + (beta*y), x = +0.0 where lhs has
// no entry; C order when rhs's fastest axis is Axis(1), F order otherwise
template <class I, class Iptr>
Array2 add_dense_mat_same_ordering(const CsMatI<I, Iptr>& lhs, const Array2& rhs, double alpha,
                                   double beta) {
    Array2 out = sprs::detail::fastest_axis(rhs) == 1 ? Array2::zeros(rhs.rows, rhs.cols)
                                                : Array2::zeros_f(rhs.rows, rhs.cols);
    sprs::detail::binop_dense(lhs.device(), SPRS_B200_BINOP_ADD, alpha, beta, rhs, out);
    return out;
}
// mul_dense_mat_same_ordering (binop.rs:331-371): (alpha*x)*y
template <class I, class Iptr>
Array2 mul_dense_mat_same_ordering(const CsMatI<I, Iptr>& lhs, const Array2& rhs, double alpha) {
    Array2 out = sprs::detail::fastest_axis(rhs) == 1 ? Array2::zeros(rhs.rows, rhs.cols)
                                                : Array2::zeros_f(rhs.rows, rhs.cols);
    sprs::detail::binop_dense(lhs.device(), SPRS_B200_BINOP_MUL, alpha, 0.0, rhs, out);
    return out;
}
}  // namespace binop

// `&A + &D` (csmat.rs:1951-1987): A converted first when its storage does not match D's layout
template <class I, class Iptr>
Array2 operator+(const CsMatI<I, Iptr>& a, const Array2& d) {
    if (a.is_csr() == (detail::fastest_axis(d) == 1)) return binop::add_dense_mat_same_ordering(a, d, 1.0, 1.0);
    return binop::add_dense_mat_same_ordering(a.to_other_storage(), d, 1.0, 1.0);
}

// ---- bmat / vstack / hstack (construct.rs) and kronecker_product (kronecker.rs) on the device.
// Results are bit-identical to the reference; a result dimension >= 2^32 panics (device
// mirrors index with u32) even where usize would allow it.  Blocks are pointers, nullptr = None.
namespace detail {
inline sprs_b200_csmat* bmat_dev(Context& ctx, size_t n_rows, size_t n_cols,
                                 const std::vector<const sprs_b200_csmat*>& grid) {
    sprs_b200_csmat* c = nullptr;
    ctx.check(sprs_b200_csmat_bmat(ctx.handle(), n_rows, n_cols, grid.data(), &c));
    return c;
}
}  // namespace detail

// bmat: the asserts in the reference's order, then the device concatenation (always CSR)
template <class I, class Iptr>
CsMatI<I, Iptr> bmat(const std::vector<std::vector<const CsMatI<I, Iptr>*>>& blocks) {
    if (blocks.empty() || blocks[0].empty()) throw Panic("Empty stacking list");
    const size_t nbr = blocks.size(), nbc = blocks[0].size();
    for (const auto& row : blocks)
        if (row.size() != nbc) throw Panic("Dimension mismatch");
    for (const auto& row : blocks) {
        bool any = false;
        for (const auto* m : row) any = any || m;
        if (!any) throw Panic("Empty bmat row");
    }
    std::vector<size_t> widths(nbc, 0);
    for (size_t j = 0; j < nbc; ++j) {
        bool any = false;
        for (const auto& row : blocks)
            if (row[j]) {
                any = true;
                widths[j] = std::max(widths[j], row[j]->cols());
            }
        if (!any) throw Panic("Empty bmat col");
    }
    Context& ctx = Context::thread_default();
    std::vector<const sprs_b200_csmat*> grid;
    size_t rows = 0, cols = 0;
    for (size_t i = 0; i < nbr; ++i) {
        size_t height = 0;
        for (size_t j = 0; j < nbc; ++j) {
            const auto* m = blocks[i][j];
            grid.push_back(m ? m->device() : nullptr);
            if (m) height = std::max(height, m->rows());
            if (i == 0) cols += m ? m->cols() : widths[j];
        }
        rows += height;
    }
    sprs_b200_csmat* c = detail::bmat_dev(ctx, nbr, nbc, grid);
    CsMatI<I, Iptr> out = CsMatI<I, Iptr>::download(ctx, c, CSR, rows, cols);
    sprs_b200_csmat_free(c);
    return out;
}

// vstack: the CSR forms stacked vertically (always CSR)
template <class I, class Iptr>
CsMatI<I, Iptr> vstack(const std::vector<CsMatI<I, Iptr>>& mats) {
    if (mats.empty()) throw Panic("Empty stacking list");
    std::vector<std::vector<const CsMatI<I, Iptr>*>> col;
    for (const auto& m : mats) col.push_back({&m});
    return bmat(col);
}

// hstack: the CSC forms stacked horizontally (always CSC) -- on the device, the vstack of the
// blocks' transpose views, read back as the CSC it is
template <class I, class Iptr>
CsMatI<I, Iptr> hstack(const std::vector<CsMatI<I, Iptr>>& mats) {
    if (mats.empty()) throw Panic("Empty stacking list");
    Context& ctx = Context::thread_default();
    std::vector<const sprs_b200_csmat*> views;
    size_t cols = 0;
    int st = SPRS_B200_OK;
    for (const auto& m : mats) {
        sprs_b200_csmat* v = nullptr;
        if ((st = sprs_b200_csmat_transpose_view(ctx.handle(), m.device(), &v)) != SPRS_B200_OK)
            break;
        views.push_back(v);
        cols += m.cols();
    }
    sprs_b200_csmat* c = nullptr;
    if (st == SPRS_B200_OK) st = sprs_b200_csmat_bmat(ctx.handle(), views.size(), 1, views.data(), &c);
    for (const auto* v : views) sprs_b200_csmat_free(const_cast<sprs_b200_csmat*>(v));
    ctx.check(st);
    CsMatI<I, Iptr> out = CsMatI<I, Iptr>::download(ctx, c, CSC, mats[0].rows(), cols);
    sprs_b200_csmat_free(c);
    return out;
}

// kronecker_product: in a's storage, b converted when the storages differ.  A produced index
// that does not fit I panics like the reference's `I::from(..).unwrap()`.
template <class I, class Iptr>
CsMatI<I, Iptr> kronecker_product(const CsMatI<I, Iptr>& a, const CsMatI<I, Iptr>& b) {
    if (a.nnz() && b.nnz()) {
        auto max_inner = [&](const CsMatI<I, Iptr>& m) -> uint64_t {  // in a's storage
            uint64_t top = 0;
            for (size_t o = 0; o < m.outer_dims(); ++o)
                if (m.indptr()[o + 1] > m.indptr()[o])
                    top = m.storage() == a.storage()
                              ? std::max<uint64_t>(top, (uint64_t)m.indices()[(size_t)(m.indptr()[o + 1] - m.indptr()[0]) - 1])
                              : o;
            return top;
        };
        const uint64_t inner_b = b.storage() == a.storage() ? b.inner_dims() : b.outer_dims();
        const unsigned __int128 top = (unsigned __int128)max_inner(a) * inner_b + max_inner(b);
        if (top > (unsigned __int128)(uint64_t)std::numeric_limits<I>::max())
            throw Panic("called `Option::unwrap()` on a `None` value");
    }
    Context& ctx = Context::thread_default();
    sprs_b200_csmat* c = nullptr;
    ctx.check(sprs_b200_csmat_kron(ctx.handle(), a.device(), b.device(), &c));
    CsMatI<I, Iptr> out = CsMatI<I, Iptr>::download(ctx, c, a.storage(), a.rows() * b.rows(),
                                                    a.cols() * b.cols());
    sprs_b200_csmat_free(c);
    return out;
}

// `&A * &x`, x: Array1 (csmat.rs:2119-2160)
template <class I, class Iptr>
Array1 operator*(const CsMatI<I, Iptr>& a, const Array1& x) {
    if (a.cols() != x.size()) throw Panic("Dimension mismatch");
    Array1 y(a.rows(), 0.0);
    Context& ctx = Context::thread_default();
    ctx.check(sprs_b200_mul_mat_vec(ctx.handle(), a.device(), x.data(), x.size(), y.data(), y.size()));
    return y;
}
// `&A * &B`, B: Array2 (csmat.rs:1989-2048): k >= 8 -> rowmaj kernel / C order
template <class I, class Iptr>
Array2 operator*(const CsMatI<I, Iptr>& a, const Array2& b) {
    const size_t rows = a.rows(), cols = b.cols;
    if (cols >= 8) {
        Array2 res = Array2::zeros(rows, cols);
        if (a.is_csr()) prod::csr_mulacc_dense_rowmaj(a, b, res);
        else prod::csc_mulacc_dense_rowmaj(a, b, res);
        return res;
    }
    Array2 res = Array2::zeros_f(rows, cols);
    if (a.is_csr()) prod::csr_mulacc_dense_colmaj(a, b, res);
    else prod::csc_mulacc_dense_colmaj(a, b, res);
    return res;
}
// `&A * &v`, v: CsVec (vec.rs:1104-1131).  CSR: prod::csr_mul_csvec (prod.rs:162-184), the
// per-row sorted-merge dot on the device (csrc/csvec.cu, bit-identical), exact zeros dropped
// (:178-180).  CSC: `self.mul(&rhs.col_view())`, the sparse-sparse product (vec.rs:1128).
template <class I, class Iptr>
CsVecI<I> operator*(const CsMatI<I, Iptr>& a, const CsVecI<I>& v) {
    if (!a.is_csr()) {
        auto col = CsMatI<I, Iptr>::new_csc({v.dim, 1}, {(Iptr)0, (Iptr)v.nnz()}, v.indices, v.data);
        auto c = (a * col).to_csc();
        return CsVecI<I>(a.rows(), c.indices(), c.data());
    }
    if (v.dim == 0) return CsVecI<I>::empty(0);
    if (a.cols() != v.dim) throw Panic("Dimension mismatch");
    Context& ctx = Context::thread_default();
    Array1 y(a.rows(), 0.0);
    ctx.check(sprs_b200_csr_mul_csvec(ctx.handle(), a.device(), v.dim, v.nnz(), v.indices.data(),
                                      (int)sizeof(I), v.data.data(), y.data(), y.size()));
    CsVecI<I> res = CsVecI<I>::empty(a.rows());
    for (size_t r = 0; r < y.size(); ++r)
        if (y[r] != 0.0) {
            res.indices.push_back((I)r);
            res.data.push_back(y[r]);
        }
    return res;
}
// Sum of v1[i] * rhs[i] over the common pattern in ascending index order (dot_acc,
// vec.rs:846-881) on the device: row_view(v1) through the merge-dot kernel (csrc/csvec.cu),
// the reference's terms in the reference's order.
// Every term is added, one by one, to `start`.
template <class I>
double merge_dot(const CsVecI<I>& v1, size_t dim, const std::vector<I>& idx,
                 const std::vector<double>& dat, double start = 0.0) {
    if (v1.nnz() == 0 || idx.empty()) return start;
    auto row = CsMatI<I, I>::new_({1, dim}, {(I)0, (I)v1.nnz()}, v1.indices, v1.data);
    Context& ctx = Context::thread_default();
    double y = start;
    ctx.check(sprs_b200_csr_mul_csvec_acc(ctx.handle(), row.device(), dim, idx.size(), idx.data(),
                                          (int)sizeof(I), dat.data(), &y, 1));
    return y;
}
// CsVecBase::dot (vec.rs:825-881) with a sparse rhs; panics if the dimensions differ
template <class I>
double dot(const CsVecI<I>& v1, const CsVecI<I>& v2) {
    if (v1.dim != v2.dim) throw Panic("Dimension mismatch");
    return merge_dot(v1, v1.dim, v2.indices, v2.data);
}
// CsVecBase::dot_dense (vec.rs:894-904): `Iterator::sum` of the products, and std's f64 sum
// folds from -0.0 (rust-lang/rust#129321), where dot with a dense rhs (dot_acc) starts from
// +0.0.  An empty vector, or one whose every product is -0.0, gives -0.0.
template <class I>
double dot_dense(const CsVecI<I>& v1, const Array1& rhs) {
    if (v1.dim != rhs.size()) throw Panic("Dimension mismatch");
    std::vector<I> all(rhs.size());
    for (size_t i = 0; i < all.size(); ++i) all[i] = (I)i;
    return merge_dot(v1, v1.dim, all, std::vector<double>(rhs.data(), rhs.data() + rhs.size()),
                     -0.0);
}
namespace prod {
// prod::csvec_dot_by_binary_search (prod.rs:13-72): the same sum (matching entries in
// ascending index order); the reference does not compare the dimensions here.
template <class I>
double csvec_dot_by_binary_search(const CsVecI<I>& vec1, const CsVecI<I>& vec2) {
    return merge_dot(vec1, vec1.dim > vec2.dim ? vec1.dim : vec2.dim, vec2.indices, vec2.data);
}
}  // namespace prod
// `&v * &A` = row_view(v) * A (vec.rs:1084-1102)
template <class I, class Iptr>
CsVecI<I> operator*(const CsVecI<I>& v, const CsMatI<I, Iptr>& a) {
    auto row = CsMatI<I, Iptr>::new_({1, v.dim}, {(Iptr)0, (Iptr)v.nnz()}, v.indices, v.data);
    auto c = (row * a).to_csr();
    return CsVecI<I>(a.cols(), c.indices(), c.data());
}

// ------------------------------------------------------------------------------------
// sprs::linalg::bicgstab::BiCGSTAB<f64> (linalg/bicgstab.rs:95-300) with every vector
// resident on the device between iterations.  Vectors cross this API as dense Array1
// (the reference's CsVec arithmetic is dense arithmetic on the union pattern).
namespace linalg {
namespace bicgstab {
template <class I, class Iptr>
class BiCGSTAB {
   public:
    // BiCGSTAB::new (bicgstab.rs:120-146); borrows `a` like the reference's view does
    BiCGSTAB(const CsMatI<I, Iptr>& a, const Array1& x0, const Array1& b) : a_(&a) {
        if (a.cols() != x0.size() || a.rows() != b.size()) throw Panic("Dimension mismatch");
        Context& ctx = Context::thread_default();
        ctx.check(sprs_b200_bicgstab_new(ctx.handle(), a.device(), x0.data(), b.data(),
                                         b.size(), &h_));
    }
    // Operator form (sprs_b200_bicgstab_new_op): y = A x is `matvec(d_x, d_y, stream)` with
    // device pointers to n doubles, enqueued on `stream` -- a matrix-free operator or the
    // row-partitioned SpMV + all-gather of a multi-GPU caller.  a() is not available.
    using MatVec = std::function<void(const double* d_x, double* d_y, void* stream)>;
    BiCGSTAB(size_t n, MatVec matvec, const Array1& x0, const Array1& b)
        : a_(nullptr), n_(n), op_(std::make_unique<MatVec>(std::move(matvec))) {
        if (x0.size() != n || b.size() != n) throw Panic("Dimension mismatch");
        Context& ctx = Context::thread_default();
        ctx.check(sprs_b200_bicgstab_new_op(ctx.handle(), n, &BiCGSTAB::trampoline, op_.get(),
                                            x0.data(), b.data(), 0, &h_));
    }
    BiCGSTAB(const BiCGSTAB&) = delete;
    BiCGSTAB& operator=(const BiCGSTAB&) = delete;
    ~BiCGSTAB() { sprs_b200_bicgstab_free(h_); }

    // BiCGSTAB::solve (bicgstab.rs:151-175): first = true for Ok, false for Err; the
    // solver comes back either way, as in Result<Box<Self>, Box<Self>>
    static std::pair<bool, std::unique_ptr<BiCGSTAB>> solve(const CsMatI<I, Iptr>& a,
                                                            const Array1& x0, const Array1& b,
                                                            double tol, size_t max_iter) {
        auto s = std::make_unique<BiCGSTAB>(a, x0, b);
        int converged = 0;
        check(sprs_b200_bicgstab_solve(s->h_, tol, max_iter, &converged));
        return {converged != 0, std::move(s)};
    }
    double step() {
        double err = 0.0;
        check(sprs_b200_bicgstab_step(h_, &err));
        return err;
    }
    void soft_restart() { check(sprs_b200_bicgstab_soft_restart(h_)); }
    void hard_restart() { check(sprs_b200_bicgstab_hard_restart(h_)); }
    BiCGSTAB& with_restart_threshold(double thresh) {
        check(sprs_b200_bicgstab_set_restart_threshold(h_, thresh));
        return *this;
    }
    size_t iteration_count() const { return (size_t)counts()[0]; }
    size_t soft_restart_count() const { return (size_t)counts()[1]; }
    size_t hard_restart_count() const { return (size_t)counts()[2]; }
    double err() const { return scalars()[0]; }
    double rho() const { return scalars()[1]; }
    double soft_restart_threshold() const { return scalars()[2]; }
    const CsMatI<I, Iptr>& a() const { return *a_; }
    Array1 x() const { return vec(SPRS_B200_BICGSTAB_X); }
    Array1 b() const { return vec(SPRS_B200_BICGSTAB_B); }
    Array1 r() const { return vec(SPRS_B200_BICGSTAB_R); }
    Array1 rhat() const { return vec(SPRS_B200_BICGSTAB_RHAT); }
    Array1 p() const { return vec(SPRS_B200_BICGSTAB_P); }

   private:
    static void check(int st) { Context::thread_default().check(st); }
    std::array<uint64_t, 3> counts() const {
        std::array<uint64_t, 3> c{};
        check(sprs_b200_bicgstab_stats(h_, c.data(), nullptr));
        return c;
    }
    std::array<double, 3> scalars() const {
        std::array<double, 3> v{};
        check(sprs_b200_bicgstab_stats(h_, nullptr, v.data()));
        return v;
    }
    Array1 vec(int which) const {
        Array1 out(a_ ? a_->rows() : n_);
        check(sprs_b200_bicgstab_get(h_, which, out.data(), out.size()));
        return out;
    }
    static int trampoline(void* user, const double* d_x, double* d_y, void* stream) {
        try {
            (*static_cast<MatVec*>(user))(d_x, d_y, stream);
            return 0;
        } catch (...) {
            return 1;  // never unwind through the C frames: the call fails with a status
        }
    }
    const CsMatI<I, Iptr>* a_;
    size_t n_ = 0;
    std::unique_ptr<MatVec> op_;
    sprs_b200_bicgstab* h_ = nullptr;
};
}  // namespace bicgstab

// sprs::linalg::trisolve (linalg/trisolve.rs:30-262): L x = b / U x = b with a dense rhs solved
// in place on the device, bit-identical to the reference.  The reference's panics throw Panic
// in its order (square, then rhs.dim(), then storage); its Err(SingularMatrix) throws
// SingularMatrix, with rhs left as the reference leaves it.
struct SingularMatrix : std::runtime_error {  // LinalgError::SingularMatrix (errors.rs:59-69)
    size_t index;
    std::string reason;
    SingularMatrix(size_t i, const std::string& r)
        : std::runtime_error("Singular matrix at index " + std::to_string(i) + " (" + r + ")"),
          index(i), reason(r) {}
};
namespace trisolve {
namespace detail {
template <class I, class Iptr>
void solve(const CsMatI<I, Iptr>& mat, Array1& rhs, int tri, bool csr) {
    if (mat.rows() != mat.cols()) throw Panic("Non square matrix passed to solver");
    if (mat.cols() != rhs.size()) throw Panic("Dimension mismatch");
    if (mat.is_csr() != csr) throw Panic("Storage mismatch");
    Context& ctx = Context::thread_default();
    sprs_b200_trisolve* plan = nullptr;
    ctx.check(sprs_b200_trisolve_plan(ctx.handle(), mat.device(), tri, &plan));
    const int st = sprs_b200_trisolve_solve(plan, rhs.data(), rhs.size());
    uint64_t index = 0;
    int reason = 0;
    const bool singular = sprs_b200_trisolve_singular(plan, &index, &reason) != 0;
    sprs_b200_trisolve_free(plan);
    if (st == SPRS_B200_ERR_SINGULAR && singular) {
        static const char* reasons[] = {"diagonal element is 0", "diagonal element is a numeric 0",
                                        "diagonal element is a structural 0"};
        throw SingularMatrix((size_t)index, reasons[reason]);
    }
    ctx.check(st);
}
}  // namespace detail
template <class I, class Iptr>
void lsolve_csr_dense_rhs(const CsMatI<I, Iptr>& lower_tri_mat, Array1& rhs) {
    detail::solve(lower_tri_mat, rhs, SPRS_B200_TRI_LOWER, true);
}
template <class I, class Iptr>
void usolve_csr_dense_rhs(const CsMatI<I, Iptr>& upper_tri_mat, Array1& rhs) {
    detail::solve(upper_tri_mat, rhs, SPRS_B200_TRI_UPPER, true);
}
template <class I, class Iptr>
void lsolve_csc_dense_rhs(const CsMatI<I, Iptr>& lower_tri_mat, Array1& rhs) {
    detail::solve(lower_tri_mat, rhs, SPRS_B200_TRI_LOWER, false);
}
template <class I, class Iptr>
void usolve_csc_dense_rhs(const CsMatI<I, Iptr>& upper_tri_mat, Array1& rhs) {
    detail::solve(upper_tri_mat, rhs, SPRS_B200_TRI_UPPER, false);
}
}  // namespace trisolve

// sprs::linalg::diag_solve (sparse/linalg.rs): x_i /= diag_i on the device
inline void diag_solve(const Array1& diag, Array1& x) {
    if (diag.size() != x.size()) throw Panic("assertion `left == right` failed");
    Context& ctx = Context::thread_default();
    ctx.check(sprs_b200_diag_solve(ctx.handle(), diag.data(), x.data(), x.size()));
}
}  // namespace linalg

// The sprs-ldl crate (sprs-ldl/src/lib.rs): L D L^T = P A P^T on the device with the permutation
// given (new_perm) or the identity (new_), bit-identical L, D, x and singular index.  No
// fill-reducing ordering is computed.  The reference's panics throw Panic in its order (square,
// symmetry, permutation); Err(SingularMatrix) throws SingularMatrix.  After an update that
// throws SingularMatrix, l, d and solve throw it too until an update succeeds; an update with
// another pattern throws Panic before any work is done and leaves the factor as it was.
namespace ldl {
using linalg::SingularMatrix;
enum class SymmetryCheck { CheckSymmetry, DontCheckSymmetry };
namespace detail {
static const char* const kNumericZero = "diagonal element is a numeric 0";
struct Handle {
    sprs_b200_ldl* h = nullptr;
    explicit Handle(sprs_b200_ldl* p) : h(p) {}
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;
    ~Handle() { sprs_b200_ldl_free(h); }
};
inline void status(Context& ctx, int st, uint64_t index) {
    if (st == SPRS_B200_ERR_NOT_SYMMETRIC) throw Panic("Matrix is not symmetric");
    if (st == SPRS_B200_ERR_SINGULAR) throw SingularMatrix((size_t)index, kNumericZero);
    if (st == SPRS_B200_ERR_STRUCTURE) throw Panic(sprs_b200_last_error(ctx.handle()));
    ctx.check(st);
}
}  // namespace detail

// sprs::is_symmetric (sparse/symmetric.rs) on the device
template <class I, class Iptr>
bool is_symmetric(const CsMatI<I, Iptr>& mat) {
    Context& ctx = Context::thread_default();
    int out = 0;
    ctx.check(sprs_b200_is_symmetric(ctx.handle(), mat.device(), &out));
    return out != 0;
}

class LdlNumeric;
class LdlSymbolic {
   public:
    template <class I, class Iptr>
    static LdlSymbolic new_(const CsMatI<I, Iptr>& mat) {
        if (mat.rows() != mat.cols()) throw Panic("assertion `left == right` failed");
        return build(mat, nullptr, SymmetryCheck::CheckSymmetry);
    }
    // perm[k] is the outer vector of mat that is row k of P A P^T
    template <class I, class Iptr>
    static LdlSymbolic new_perm(const CsMatI<I, Iptr>& mat, const std::vector<size_t>& perm,
                                SymmetryCheck check) {
        return build(mat, &perm, check);
    }
    size_t problem_size() const { return n_; }
    size_t nnz() const { return (size_t)sprs_b200_ldl_nnz(h_->h); }
    template <class I, class Iptr>
    LdlNumeric factor(const CsMatI<I, Iptr>& mat) const;

   private:
    template <class I, class Iptr>
    static LdlSymbolic build(const CsMatI<I, Iptr>& mat, const std::vector<size_t>* perm,
                             SymmetryCheck check) {
        const size_t n = mat.rows();
        if (mat.cols() != n) throw Panic("matrix should be square");
        const bool check_sym = check == SymmetryCheck::CheckSymmetry;
        std::vector<uint32_t> p;
        if (perm) {
            if (perm->size() != n) {
                if (check_sym && !is_symmetric(mat)) throw Panic("Matrix is not symmetric");
                throw Panic("assertion failed: perm_is_valid(&perm)");
            }
            for (size_t v : *perm) p.push_back(v >= n ? (uint32_t)n : (uint32_t)v);
        }
        Context& ctx = Context::thread_default();
        sprs_b200_ldl* h = nullptr;
        const int st = sprs_b200_ldl_symbolic(ctx.handle(), mat.device(), perm ? p.data() : nullptr,
                                              check_sym ? 1 : 0, &h);
        if (st == SPRS_B200_ERR_ARGUMENT) throw Panic("assertion failed: perm_is_valid(&perm)");
        if (st == SPRS_B200_ERR_DIMENSION) throw Panic("matrix should be square");
        detail::status(ctx, st, 0);
        LdlSymbolic s;
        s.h_ = std::make_shared<detail::Handle>(h);
        s.n_ = n;
        return s;
    }
    std::shared_ptr<detail::Handle> h_;
    size_t n_ = 0;
    friend class LdlNumeric;
};

class LdlNumeric {
   public:
    template <class I, class Iptr>
    static LdlNumeric new_(const CsMatI<I, Iptr>& mat) {
        return LdlSymbolic::new_(mat).factor(mat);
    }
    template <class I, class Iptr>
    static LdlNumeric new_perm(const CsMatI<I, Iptr>& mat, const std::vector<size_t>& perm,
                               SymmetryCheck check) {
        return LdlSymbolic::new_perm(mat, perm, check).factor(mat);
    }
    template <class I, class Iptr>
    void update(const CsMatI<I, Iptr>& mat) {
        Context& ctx = Context::thread_default();
        const int st = sprs_b200_ldl_update(h_->h, mat.device());
        uint64_t index = 0;
        sprs_b200_ldl_singular(h_->h, &index);
        detail::status(ctx, st, index);
    }
    Array1 solve(const Array1& rhs) const {
        if (rhs.size() != sym_.n_) throw Panic("assertion `left == right` failed");
        Context& ctx = Context::thread_default();
        Array1 x(rhs.size());
        status(ctx, sprs_b200_ldl_solve(h_->h, rhs.data(), x.data(), x.size()));
        return x;
    }
    // L in CSC, its unit diagonal not stored
    CsMatI<size_t> l() const {
        Context& ctx = Context::thread_default();
        const size_t n = sym_.n_, nnz = this->nnz();
        std::vector<uint32_t> ip(n + 1), ind(nnz);
        std::vector<double> data(nnz);
        status(ctx, sprs_b200_ldl_get_l(h_->h, ip.data(), ind.data(), data.data()));
        return CsMatI<size_t>::new_csc({n, n}, std::vector<size_t>(ip.begin(), ip.end()),
                                       std::vector<size_t>(ind.begin(), ind.end()), std::move(data));
    }
    Array1 d() const {
        Context& ctx = Context::thread_default();
        Array1 out(sym_.n_);
        status(ctx, sprs_b200_ldl_get_d(h_->h, out.data(), out.size()));
        return out;
    }
    size_t problem_size() const { return sym_.n_; }
    size_t nnz() const { return sym_.nnz(); }

   private:
    void status(Context& ctx, int st) const {
        uint64_t index = 0;
        sprs_b200_ldl_singular(h_->h, &index);
        detail::status(ctx, st, index);
    }
    LdlSymbolic sym_;                     // the numeric handle borrows it: destroyed after h_
    std::shared_ptr<detail::Handle> h_;
    friend class LdlSymbolic;
};

template <class I, class Iptr>
LdlNumeric LdlSymbolic::factor(const CsMatI<I, Iptr>& mat) const {
    if (n_ <= 1) throw Panic("assertion failed: n > 1");  // DStack::with_capacity(n)
    Context& ctx = Context::thread_default();
    sprs_b200_ldl* h = nullptr;
    const int st = sprs_b200_ldl_factor(h_->h, mat.device(), &h);
    LdlNumeric num;
    num.sym_ = *this;
    if (h) num.h_ = std::make_shared<detail::Handle>(h);
    uint64_t index = 0;
    if (h) sprs_b200_ldl_singular(h, &index);
    detail::status(ctx, st, index);
    return num;
}
}  // namespace ldl

}  // namespace sprs
