// spmm.cu -- CSR x dense row-major matrix for sm_90a (H100).
//
// Replaces prod::csr_mulacc_dense_rowmaj (sprs/src/sparse/prod.rs:189-214), the
// kernel `&A * &B` picks when B has >= 8 columns (sprs/src/sparse/csmat.rs:2009-2018):
//     out[i,:] += sum_j A[i,j] * B[j,:]        (k-wide axpy per non-zero)
// B and C are C-order with leading dimensions ldb / ldc.
//
// One warp owns one row of A and a panel of up to 32*KV output columns; the row's
// (index, value) pairs are read coalesced 32 at a time and broadcast with shuffles,
// every lane gathers its slice of the B row (a 512-byte row at k = 64 is two fully
// coalesced 256-byte requests per non-zero) and keeps KV accumulators in registers;
// C is written exactly once.  Each output element is the sequential, unfused sum in
// storage order (mul_acc.rs:28-30), so results are bit-identical to the reference.
//
// Compulsory bytes: 12*nnz + 8*k*(cols + rows); the B-row gathers (8*k per nnz) are
// served by L2 / HBM depending on B's size (DESIGN.md "SpMM").

#include <cstdlib>

#include "common.cuh"

namespace {

constexpr int SPMM_NT = 256;

template <typename P, int KV>
__global__ void __launch_bounds__(SPMM_NT)
    spmm_rowmaj_kernel(const P* __restrict__ indptr, const uint32_t* __restrict__ indices,
                       const double* __restrict__ data, const double* __restrict__ B,
                       uint64_t ldb, uint32_t k, double* __restrict__ C, uint64_t ldc,
                       uint32_t rows, int accumulate) {
    const int lane = threadIdx.x & 31;
    const uint64_t warp0 = (blockIdx.x * (uint64_t)SPMM_NT + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * SPMM_NT) >> 5;
    for (uint64_t row = warp0; row < rows; row += nwarps) {
        const uint64_t s = (uint64_t)indptr[row], e = (uint64_t)indptr[row + 1];
        double* crow = C + row * ldc;
        for (uint32_t c0 = 0; c0 < k; c0 += 32 * KV) {
            double acc[KV];
#pragma unroll
            for (int q = 0; q < KV; ++q) {
                const uint32_t c = c0 + lane + 32 * q;
                acc[q] = (accumulate && c < k) ? crow[c] : 0.0;
            }
            for (uint64_t kk = s; kk < e; kk += 32) {
                const bool in = kk + lane < e;
                const uint32_t my_idx = in ? indices[kk + lane] : 0u;
                const double my_val = in ? data[kk + lane] : 0.0;
                const int n = (e - kk) < 32 ? (int)(e - kk) : 32;
                for (int j = 0; j < n; ++j) {
                    const uint32_t col = __shfl_sync(0xffffffffu, my_idx, j);
                    const double v = __shfl_sync(0xffffffffu, my_val, j);
                    const double* brow = B + (uint64_t)col * ldb;
#pragma unroll
                    for (int q = 0; q < KV; ++q) {
                        const uint32_t c = c0 + lane + 32 * q;
                        if (c < k) acc[q] = __dadd_rn(acc[q], __dmul_rn(v, __ldg(brow + c)));
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < KV; ++q) {
                const uint32_t c = c0 + lane + 32 * q;
                if (c < k) crow[c] = acc[q];
            }
        }
    }
}

// Vector flavour (B and C 16-byte aligned, even leading dimensions and k): lane L owns the
// column PAIRS 2L + 64 q of the panel, a 512-byte B row at k = 64 is ONE 128-bit request per lane,
// and the B rows of U consecutive non-zeros are in flight before the first product is added (in
// storage order, so the sums are the same bits).  The scalar kernel above issues one 8-byte
// load per non-zero and column and waits for it: two requests in flight per warp, bound by
// exposed DRAM latency.
template <typename P, int KV2, int U>
__global__ void __launch_bounds__(SPMM_NT)
    spmm_rowmaj_vec_kernel(const P* __restrict__ indptr, const uint32_t* __restrict__ indices,
                           const double* __restrict__ data, const double* __restrict__ B,
                           uint64_t ldb, uint32_t k, double* __restrict__ C, uint64_t ldc,
                           uint32_t rows, int accumulate) {
    const int lane = threadIdx.x & 31;
    const uint64_t warp0 = (blockIdx.x * (uint64_t)SPMM_NT + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * SPMM_NT) >> 5;
    for (uint64_t row = warp0; row < rows; row += nwarps) {
        const uint64_t s = (uint64_t)indptr[row], e = (uint64_t)indptr[row + 1];
        double* crow = C + row * ldc;
        for (uint32_t c0 = 0; c0 < k; c0 += 64 * KV2) {
            double2 acc[KV2];
#pragma unroll
            for (int q = 0; q < KV2; ++q) {
                const uint32_t c = c0 + 2 * lane + 64 * q;
                acc[q] = (accumulate && c < k) ? *(const double2*)(crow + c) : make_double2(0.0, 0.0);
            }
            for (uint64_t kk = s; kk < e; kk += 32) {
                const bool in = kk + lane < e;
                const uint32_t my_idx = in ? indices[kk + lane] : 0u;
                const double my_val = in ? data[kk + lane] : 0.0;
                const int n = (e - kk) < 32 ? (int)(e - kk) : 32;
                for (int j = 0; j < n; j += U) {
                    double v[U];
                    double2 b[U][KV2];
#pragma unroll
                    for (int u = 0; u < U; ++u) {  // all loads of U non-zeros first
                        const uint32_t col = __shfl_sync(0xffffffffu, my_idx, (j + u) & 31);
                        v[u] = __shfl_sync(0xffffffffu, my_val, (j + u) & 31);
                        const double* brow = B + (uint64_t)col * ldb;
#pragma unroll
                        for (int q = 0; q < KV2; ++q) {
                            const uint32_t c = c0 + 2 * lane + 64 * q;
                            b[u][q] = (j + u < n && c < k) ? __ldg((const double2*)(brow + c))
                                                           : make_double2(0.0, 0.0);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u)  // then the sums, in storage order
                        if (j + u < n) {
#pragma unroll
                            for (int q = 0; q < KV2; ++q) {
                                acc[q].x = __dadd_rn(acc[q].x, __dmul_rn(v[u], b[u][q].x));
                                acc[q].y = __dadd_rn(acc[q].y, __dmul_rn(v[u], b[u][q].y));
                            }
                        }
                }
            }
#pragma unroll
            for (int q = 0; q < KV2; ++q) {
                const uint32_t c = c0 + 2 * lane + 64 * q;
                if (c < k) *(double2*)(crow + c) = acc[q];
            }
        }
    }
}

}  // namespace

int spmm_rowmaj_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_b,
                       uint64_t ldb, uint64_t k, double* d_c, uint64_t ldc, int accumulate,
                       cudaStream_t s) {
    if (m->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch: spmm needs a CSR mirror");
    if (m->rows == 0 || k == 0) return SPRS_B200_OK;
    if (k > 0xffffffffull) SPRS_FAIL(ctx, SPRS_B200_ERR_UNSUPPORTED, "k too large");
    const uint64_t warps_needed = m->rows;
    uint64_t blocks = (warps_needed * 32 + SPMM_NT - 1) / SPMM_NT;
    const uint64_t cap = (uint64_t)ctx->sm_count * 64;
    if (blocks > cap) blocks = cap;
    const unsigned grid = (unsigned)blocks;
    // 128-bit flavour when every B / C row segment a lane touches is 16-byte aligned
    const bool vec = (k % 2 == 0) && (ldb % 2 == 0) && (ldc % 2 == 0) &&
                     (((uintptr_t)d_b | (uintptr_t)d_c) & 15) == 0;
#define SPMM_LAUNCH(P)                                                                        \
    do {                                                                                      \
        if (vec && k <= 64)                                                                   \
            spmm_rowmaj_vec_kernel<P, 1, 4><<<grid, SPMM_NT, 0, s>>>(                         \
                (const P*)m->d_indptr, m->d_indices, m->d_data, d_b, ldb, (uint32_t)k, d_c,   \
                ldc, (uint32_t)m->rows, accumulate);                                          \
        else if (vec)                                                                         \
            spmm_rowmaj_vec_kernel<P, 2, 2><<<grid, SPMM_NT, 0, s>>>(                         \
                (const P*)m->d_indptr, m->d_indices, m->d_data, d_b, ldb, (uint32_t)k, d_c,   \
                ldc, (uint32_t)m->rows, accumulate);                                          \
        else if (k <= 32)                                                                     \
            spmm_rowmaj_kernel<P, 1><<<grid, SPMM_NT, 0, s>>>(                                \
                (const P*)m->d_indptr, m->d_indices, m->d_data, d_b, ldb, (uint32_t)k, d_c,   \
                ldc, (uint32_t)m->rows, accumulate);                                          \
        else                                                                                  \
            spmm_rowmaj_kernel<P, 2><<<grid, SPMM_NT, 0, s>>>(                                \
                (const P*)m->d_indptr, m->d_indices, m->d_data, d_b, ldb, (uint32_t)k, d_c,   \
                ldc, (uint32_t)m->rows, accumulate);                                          \
    } while (0)
    if (m->indptr_bytes == 4)
        SPMM_LAUNCH(uint32_t);
    else
        SPMM_LAUNCH(uint64_t);
#undef SPMM_LAUNCH
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}
