// csvec.cu -- CSR matrix x SPARSE vector for sm_90a (H100).
//
// Replaces prod::csr_mul_csvec (sprs/src/sparse/prod.rs:162-184), what `&A * &v` runs for a
// CSR matrix and a CsVec (sprs/src/sparse/vec.rs:1104-1131) -- the README example and
// BASELINE config 1 (sprs/src/lib.rs:54-60).  Row i of the result is the reference's
// sorted-merge dot product (CsVecBase::dot_acc, vec.rs:846-881): ONLY the entries present in
// both patterns are multiplied, and they are summed sequentially in ascending column order.
// An A entry opposite a structural zero of v takes no part at all, so an Inf/NaN stored in A
// there does not poison the row (a dense x with explicit zeros would give Inf*0 = NaN).
//
// Device form: v is scattered into a dense value array plus a presence byte per column (both
// scratch, cols entries); one warp owns one row, reads 32 (index, value) pairs coalesced,
// gathers presence and value, and the products of the lanes that hit are added ONE AT A TIME
// in lane order (ballot + shuffle), every lane carrying the same running sum.  That is the
// reference's order exactly: results are bit-identical, whatever the values.  Not a
// bandwidth path (config 1 is the plumbing case); rows are independent, y is written once.
#include "common.cuh"

namespace {

constexpr int CSVEC_NT = 256;

template <typename I>
__global__ void __launch_bounds__(CSVEC_NT)
    csvec_scatter_kernel(const I* __restrict__ v_indices, const double* __restrict__ v_data,
                         uint64_t v_nnz, double* __restrict__ x, unsigned char* __restrict__ present) {
    const uint64_t i = blockIdx.x * (uint64_t)CSVEC_NT + threadIdx.x;
    if (i >= v_nnz) return;
    const uint64_t c = (uint64_t)v_indices[i];
    x[c] = v_data[i];
    present[c] = 1;
}

template <typename P>
__global__ void __launch_bounds__(CSVEC_NT)
    csr_mul_csvec_kernel(const P* __restrict__ indptr, const uint32_t* __restrict__ indices,
                         const double* __restrict__ data, const double* __restrict__ x,
                         const unsigned char* __restrict__ present, double* __restrict__ y,
                         uint64_t rows) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const uint64_t warp0 = (blockIdx.x * (uint64_t)CSVEC_NT + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * CSVEC_NT) >> 5;
    for (uint64_t row = warp0; row < rows; row += nwarps) {
        const uint64_t s = (uint64_t)indptr[row], e = (uint64_t)indptr[row + 1];
        double acc = 0.0;  // N::zero(), identical in every lane
        for (uint64_t k = s; k < e; k += 32) {
            bool hit = false;
            double prod = 0.0;
            if (k + lane < e) {
                const uint32_t c = indices[k + lane];
                hit = present[c] != 0;
                if (hit) prod = __dmul_rn(data[k + lane], x[c]);  // a * b, then the add below
            }
            unsigned m = __ballot_sync(FULL, hit);
            while (m) {  // sum.mul_acc(left_val, right_val) in ascending column order
                const int j = __ffs(m) - 1;
                m &= m - 1;
                acc = __dadd_rn(acc, __shfl_sync(FULL, prod, j));
            }
        }
        if (lane == 0) y[row] = acc;
    }
}

}  // namespace

int sprs_b200_csr_mul_csvec(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, uint64_t dim,
                            uint64_t v_nnz, const void* v_indices, int index_bytes,
                            const double* v_data, double* res, uint64_t res_len) {
    if (!ctx || !mat) return SPRS_B200_ERR_ARGUMENT;
    // assert_eq!(lhs.cols(), rhs.dim(), "Dimension mismatch")  prod.rs:174
    if (mat->cols != dim || mat->rows != res_len)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (mat->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch: csr_mul_csvec needs a CSR mirror");
    if (index_bytes != 4 && index_bytes != 8)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "index width must be 4 or 8 bytes");
    if ((v_nnz && (!v_indices || !v_data)) || (res_len && !res)) return SPRS_B200_ERR_ARGUMENT;
    if (v_nnz > dim) SPRS_FAIL(ctx, SPRS_B200_ERR_STRUCTURE, "sparse vector has more entries than its dimension");
    if (res_len == 0) return SPRS_B200_OK;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    // the CsVec invariant (indices < dim) is the caller's, like every structure check
    // (SURVEY 8b); verify it here anyway -- an out-of-range index would be a wild store
    for (uint64_t i = 0; i < v_nnz; ++i) {
        const uint64_t c = index_bytes == 4 ? ((const uint32_t*)v_indices)[i]
                                            : ((const uint64_t*)v_indices)[i];
        if (c >= dim) SPRS_FAIL(ctx, SPRS_B200_ERR_STRUCTURE, "sparse vector index out of bounds");
    }
    void *d_x = nullptr, *d_y = nullptr, *d_v = nullptr, *d_present = nullptr;
    const size_t v_bytes = (size_t)v_nnz * (8 + (size_t)index_bytes);
    SPRS_TRY(ctx_scratch(ctx, 1, dim * sizeof(double), &d_x));
    SPRS_TRY(ctx_scratch(ctx, 2, res_len * sizeof(double), &d_y));
    SPRS_TRY(ctx_scratch(ctx, 3, v_bytes + 16, &d_v));
    SPRS_TRY(ctx_scratch(ctx, 0, dim, &d_present));
    // values first (8-byte aligned), then the indices
    double* d_vdata = (double*)d_v;
    void* d_vind = (unsigned char*)d_v + (size_t)v_nnz * 8;
    if (dim) {
        SPRS_CUDA(ctx, cudaMemsetAsync(d_present, 0, dim, s));
        // x needs no clearing: entries without a presence mark are never read
    }
    if (v_nnz) {
        SPRS_CUDA(ctx, cudaMemcpyAsync(d_vdata, v_data, v_nnz * 8, cudaMemcpyHostToDevice, s));
        SPRS_CUDA(ctx, cudaMemcpyAsync(d_vind, v_indices, v_nnz * (size_t)index_bytes,
                                       cudaMemcpyHostToDevice, s));
        const unsigned grid = (unsigned)((v_nnz + CSVEC_NT - 1) / CSVEC_NT);
        if (index_bytes == 4)
            csvec_scatter_kernel<uint32_t><<<grid, CSVEC_NT, 0, s>>>(
                (const uint32_t*)d_vind, d_vdata, v_nnz, (double*)d_x, (unsigned char*)d_present);
        else
            csvec_scatter_kernel<uint64_t><<<grid, CSVEC_NT, 0, s>>>(
                (const uint64_t*)d_vind, d_vdata, v_nnz, (double*)d_x, (unsigned char*)d_present);
        ctx->launches += 1;
    }
    uint64_t blocks = (res_len * 32 + CSVEC_NT - 1) / CSVEC_NT;
    const uint64_t cap = (uint64_t)ctx->sm_count * 32;
    if (blocks > cap) blocks = cap;
    if (mat->indptr_bytes == 4)
        csr_mul_csvec_kernel<uint32_t><<<(unsigned)blocks, CSVEC_NT, 0, s>>>(
            (const uint32_t*)mat->d_indptr, mat->d_indices, mat->d_data, (const double*)d_x,
            (const unsigned char*)d_present, (double*)d_y, res_len);
    else
        csr_mul_csvec_kernel<uint64_t><<<(unsigned)blocks, CSVEC_NT, 0, s>>>(
            (const uint64_t*)mat->d_indptr, mat->d_indices, mat->d_data, (const double*)d_x,
            (const unsigned char*)d_present, (double*)d_y, res_len);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    SPRS_CUDA(ctx, cudaMemcpyAsync(res, d_y, res_len * sizeof(double), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    return SPRS_B200_OK;
}
