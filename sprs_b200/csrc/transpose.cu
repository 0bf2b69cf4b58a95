// transpose.cu -- storage and format conversions on the device: CSR <-> CSC, COO -> CSR
// (triplets) and the dense boundary (to_dense, from_dense and the sparse (+) dense binops, which
// share the to_dense kernel; section at the end of the file).
//
// CSR <-> CSC:
// Replaces CsMatBase::to_other_storage / raw::convert_mat_storage
// (sprs/src/sparse/csmat.rs:1405-1426, 1782-1829): a counting sort of the non-zeros
// by inner index that keeps the outer order inside every bucket, so the result has
// ascending indices per outer dimension (the reference walks outer dims in order,
// csmat.rs:1814-1822).  It is what lets CSC operands use the CSR kernels:
// `csc_mulacc_*` and `mul_acc_mat_vec_csc` (prod.rs:74-99, 219-269) accumulate each
// output element in ascending column order, exactly the order the CSR kernels use on
// the converted matrix.
//
// Device algorithm: stable LSD radix sort of (inner index, source position) pairs,
// 8 bits per pass (ceil(log2(inner)/8) passes), then one gather pass writes
// out_indices[i] = outer(pos) (binary search in indptr) and out_data[i] = data[pos].
// A pass = per-block digit histograms -> device scan -> stable scatter (per-warp
// match_any ranking keeps equal keys in source order).  Deterministic, no atomics on
// the payload.  HBM-bound: 8 B read + 8 B write per non-zero per pass.

#include "common.cuh"
#include "scan.cuh"

#include <cmath>

namespace {

constexpr int RS_NT = 256;
constexpr int RS_IPT = 16;                 // items per thread
constexpr int RS_CHUNK = RS_NT * RS_IPT;   // 4096 items per block
constexpr int RS_WARPS = RS_NT / 32;
constexpr int RS_WCHUNK = RS_CHUNK / RS_WARPS;  // contiguous items per warp (512)

// pass 0 reads keys straight from `indices` and uses pos = position
__global__ void __launch_bounds__(RS_NT)
    rs_hist_kernel(const uint32_t* __restrict__ keys, uint64_t n, int shift,
                   uint32_t* __restrict__ hist /* [256][nblocks] */, uint32_t nblocks) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t base = (uint64_t)blockIdx.x * RS_CHUNK;
#pragma unroll
    for (int i = 0; i < RS_IPT; ++i) {
        const uint64_t j = base + threadIdx.x + (uint64_t)i * RS_NT;
        if (j < n) atomicAdd(&h[(keys[j] >> shift) & 255u], 1u);
    }
    __syncthreads();
    hist[(uint64_t)threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x];
}

__global__ void __launch_bounds__(RS_NT)
    rs_scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ pos_in,
                      uint64_t n, int shift, const uint64_t* __restrict__ offsets /* scanned */,
                      uint32_t nblocks, uint32_t* __restrict__ keys_out,
                      uint32_t* __restrict__ pos_out) {
    __shared__ uint32_t wh[RS_WARPS][256];   // per-warp digit counters / running offsets
    __shared__ uint64_t gbase[256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < RS_WARPS * 256; i += RS_NT) (&wh[0][0])[i] = 0;
    gbase[threadIdx.x] = offsets[(uint64_t)threadIdx.x * nblocks + blockIdx.x];
    __syncthreads();
    // each warp owns a CONTIGUOUS run of the block's items, visited row by row (32 at a time)
    const uint64_t wbase = (uint64_t)blockIdx.x * RS_CHUNK + (uint64_t)warp * RS_WCHUNK;
    uint32_t key[RS_IPT], pos[RS_IPT];
#pragma unroll
    for (int i = 0; i < RS_IPT; ++i) {
        const uint64_t j = wbase + (uint64_t)i * 32 + lane;
        const bool in = j < n;
        key[i] = in ? keys_in[j] : 0xffffffffu;
        pos[i] = in ? (pos_in ? pos_in[j] : (uint32_t)j) : 0u;
        const uint32_t d = (key[i] >> shift) & 255u;
        const uint32_t peers = __match_any_sync(0xffffffffu, in ? d : 256u + lane);
        if (in && lane == __ffs(peers) - 1) wh[warp][d] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    {   // exclusive scan over warps for digit = threadIdx.x, seeded with the global offset
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) {
            const uint32_t c = wh[w][threadIdx.x];
            wh[w][threadIdx.x] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < RS_IPT; ++i) {
        const uint64_t j = wbase + (uint64_t)i * 32 + lane;
        const bool in = j < n;
        const uint32_t d = (key[i] >> shift) & 255u;
        const uint32_t peers = __match_any_sync(0xffffffffu, in ? d : 256u + lane);
        uint32_t off = 0;
        if (in) off = wh[warp][d] + __popc(peers & ((1u << lane) - 1u));
        __syncwarp();
        if (in && lane == __ffs(peers) - 1) wh[warp][d] += __popc(peers);
        __syncwarp();
        if (in) {
            const uint64_t dst = gbase[d] + off;
            keys_out[dst] = key[i];
            pos_out[dst] = pos[i];
        }
    }
}

__global__ void count_inner_kernel(const uint32_t* __restrict__ indices, uint64_t nnz,
                                   uint32_t* __restrict__ counts) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < nnz) atomicAdd(&counts[indices[i]], 1u);
}

template <typename P>
__global__ void gather_transposed_kernel(const uint32_t* __restrict__ pos, uint64_t nnz,
                                         const P* __restrict__ indptr, uint32_t outer,
                                         const double* __restrict__ data,
                                         uint32_t* __restrict__ out_indices,
                                         double* __restrict__ out_data) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    const uint32_t p = pos[i];
    uint32_t lo = 0, hi = outer;  // outer index o with indptr[o] <= p < indptr[o+1]
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if ((uint64_t)indptr[(size_t)mid + 1] > p)
            hi = mid;
        else
            lo = mid + 1;
    }
    out_indices[i] = lo;
    out_data[i] = data[p];
}

template <typename TIn, typename TOut>
__global__ void narrow_kernel(const TIn* __restrict__ in, TOut* __restrict__ out, uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = (TOut)in[i];
}

inline unsigned grid_for(uint64_t n) { return (unsigned)((n + 255) / 256); }

// Stable LSD radix sort of n (key, pos) pairs on `key_bits` bits; pos_in == nullptr means
// pos = 0..n-1.  Uses the caller's ping-pong buffers; returns pointers to the sorted arrays.
struct SortBuffers {
    uint32_t *kbuf[2] = {nullptr, nullptr}, *pbuf[2] = {nullptr, nullptr}, *hist = nullptr;
    uint64_t* offs = nullptr;
    uint32_t nblocks = 0;
    int alloc(uint64_t n) {
        nblocks = (uint32_t)((n + RS_CHUNK - 1) / RS_CHUNK);
        if (cudaMalloc((void**)&kbuf[0], n * 4) != cudaSuccess ||
            cudaMalloc((void**)&kbuf[1], n * 4) != cudaSuccess ||
            cudaMalloc((void**)&pbuf[0], n * 4) != cudaSuccess ||
            cudaMalloc((void**)&pbuf[1], n * 4) != cudaSuccess ||
            cudaMalloc((void**)&hist, 256ull * nblocks * 4) != cudaSuccess ||
            cudaMalloc((void**)&offs, (256ull * nblocks + 1) * 8) != cudaSuccess)
            return SPRS_B200_ERR_CUDA;
        return SPRS_B200_OK;
    }
    void release() {
        for (int i = 0; i < 2; ++i) {
            if (kbuf[i]) cudaFree(kbuf[i]);
            if (pbuf[i]) cudaFree(pbuf[i]);
            kbuf[i] = pbuf[i] = nullptr;
        }
        if (hist) cudaFree(hist);
        if (offs) cudaFree(offs);
        hist = nullptr;
        offs = nullptr;
    }
};

int bits_for(uint64_t range) {
    int bits = 1;
    while (bits < 32 && (1ull << bits) < range) ++bits;
    return bits;
}

int stable_sort_pairs(sprs_b200_ctx* ctx, SortBuffers& b, const uint32_t* keys_in,
                      const uint32_t* pos_in, uint64_t n, int key_bits, cudaStream_t s,
                      const uint32_t** keys_out, const uint32_t** pos_out) {
    const int passes = (key_bits + 7) / 8;
    const uint32_t* kin = keys_in;
    const uint32_t* pin = pos_in;
    // never scatter into the buffer currently being read
    int w = (kin == b.kbuf[0] || pin == b.pbuf[0]) ? 1 : 0;
    for (int p = 0; p < passes; ++p) {
        rs_hist_kernel<<<b.nblocks, RS_NT, 0, s>>>(kin, n, 8 * p, b.hist, b.nblocks);
        ctx->launches += 1;
        SPRS_TRY((device_exclusive_scan<uint32_t, uint64_t>(ctx, b.hist, 256ull * b.nblocks,
                                                            b.offs, s)));
        rs_scatter_kernel<<<b.nblocks, RS_NT, 0, s>>>(kin, pin, n, 8 * p, b.offs, b.nblocks,
                                                      b.kbuf[w], b.pbuf[w]);
        ctx->launches += 1;
        kin = b.kbuf[w];
        pin = b.pbuf[w];
        w ^= 1;
    }
    *keys_out = kin;
    *pos_out = pin;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

// ---- COO -> CSR helpers (TriMatBase::to_csr, sprs/src/sparse/triplet_iter.rs:127-224)
__global__ void gather_u32_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ pos,
                                  uint64_t n, uint32_t* __restrict__ dst) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[pos[i]];
}
__global__ void head_flags_kernel(const uint32_t* __restrict__ row, const uint32_t* __restrict__ col,
                                  uint64_t n, uint32_t* __restrict__ flag) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) flag[i] = (i == 0 || row[i] != row[i - 1] || col[i] != col[i - 1]) ? 1u : 0u;
}
// one thread per run head: sums the duplicates in sorted (= insertion) order, like the
// reference's duplicate summation (triplet_iter.rs:143-176), writes the unique entry
__global__ void compress_runs_kernel(const uint32_t* __restrict__ row, const uint32_t* __restrict__ col,
                                     const uint32_t* __restrict__ pos, const uint32_t* __restrict__ flag,
                                     const uint64_t* __restrict__ uidx, const double* __restrict__ vals,
                                     uint64_t n, uint32_t* __restrict__ out_idx,
                                     double* __restrict__ out_val, uint32_t* __restrict__ row_counts) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n || !flag[i]) return;
    double sum = vals[pos[i]];
    for (uint64_t j = i + 1; j < n && !flag[j]; ++j) sum = __dadd_rn(sum, vals[pos[j]]);
    const uint64_t u = uidx[i];
    out_idx[u] = col[i];
    out_val[u] = sum;
    atomicAdd(&row_counts[row[i]], 1u);
}

}  // namespace

int transpose_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, sprs_b200_csmat* t,
                     cudaStream_t s) {
    if (m->nnz >= 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_UNSUPPORTED, "to_other_storage: nnz >= 2^32 not supported");
    // gh374 (sprs/tests/gh374.rs): the outer indices must fit the index type; device
    // mirrors use u32 indices, so only > 2^32-1 outer dims can fail.
    if (m->outer > 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE,
                  "Index type is not large enough to hold the number of rows requested");
    t->ctx = ctx;
    t->storage = m->storage == SPRS_B200_CSR ? SPRS_B200_CSC : SPRS_B200_CSR;
    t->rows = m->rows;
    t->cols = m->cols;
    t->nnz = m->nnz;
    t->outer = m->inner;
    t->inner = m->outer;
    t->indptr_bytes = 4;
    t->owns = true;
    const uint64_t nnz = m->nnz, inner = m->inner;
    SPRS_CUDA(ctx, cudaMalloc(&t->d_indptr, (inner + 1) * sizeof(uint32_t) + 16));
    SPRS_CUDA(ctx, cudaMalloc((void**)&t->d_indices, nnz * sizeof(uint32_t) + 16));
    SPRS_CUDA(ctx, cudaMalloc((void**)&t->d_data, nnz * sizeof(double) + 16));

    // ---- new indptr: histogram of inner indices + exclusive scan
    uint32_t* counts = nullptr;
    uint64_t* ip64 = nullptr;
    SPRS_CUDA(ctx, cudaMalloc((void**)&counts, (inner + 1) * sizeof(uint32_t)));
    SPRS_CUDA(ctx, cudaMalloc((void**)&ip64, (inner + 1) * sizeof(uint64_t)));
    int st = SPRS_B200_OK;
    SortBuffers sb;
    do {
        cudaError_t e = cudaMemsetAsync(counts, 0, (inner + 1) * sizeof(uint32_t), s);
        if (e != cudaSuccess) { st = SPRS_B200_ERR_CUDA; break; }
        if (nnz) {
            count_inner_kernel<<<grid_for(nnz), 256, 0, s>>>(m->d_indices, nnz, counts);
            ctx->launches += 1;
        }
        if ((st = device_exclusive_scan<uint32_t, uint64_t>(ctx, counts, inner, ip64, s)) !=
            SPRS_B200_OK)
            break;
        narrow_kernel<uint64_t, uint32_t><<<grid_for(inner + 1), 256, 0, s>>>(
            ip64, (uint32_t*)t->d_indptr, inner + 1);
        ctx->launches += 1;
        if (nnz == 0) break;

        // ---- stable LSD radix sort of (inner index, position)
        if ((st = sb.alloc(nnz)) != SPRS_B200_OK) {
            sprs_b200_set_error(ctx, "to_other_storage: cudaMalloc failed");
            break;
        }
        const uint32_t *kin = nullptr, *pin = nullptr;
        if ((st = stable_sort_pairs(ctx, sb, m->d_indices, nullptr, nnz, bits_for(inner), s, &kin,
                                    &pin)) != SPRS_B200_OK)
            break;
        if (m->indptr_bytes == 4)
            gather_transposed_kernel<uint32_t><<<grid_for(nnz), 256, 0, s>>>(
                pin, nnz, (const uint32_t*)m->d_indptr, (uint32_t)m->outer, m->d_data,
                t->d_indices, t->d_data);
        else
            gather_transposed_kernel<uint64_t><<<grid_for(nnz), 256, 0, s>>>(
                pin, nnz, (const uint64_t*)m->d_indptr, (uint32_t)m->outer, m->d_data,
                t->d_indices, t->d_data);
        ctx->launches += 1;
    } while (0);
    cudaError_t e = cudaStreamSynchronize(s);
    if (st == SPRS_B200_OK && e == cudaSuccess) e = cudaGetLastError();
    if (st == SPRS_B200_OK && e != cudaSuccess) {
        sprs_b200_set_error(ctx, cudaGetErrorString(e));
        st = SPRS_B200_ERR_CUDA;
    }
    cudaFree(counts);
    cudaFree(ip64);
    sb.release();
    return st;
}

// COO (device arrays, any order, duplicates allowed) -> CSR mirror with ascending unique
// column indices per row and duplicates summed: TriMatBase::to_csr
// (sprs/src/sparse/triplet_iter.rs:127-224).  Two stable radix sorts (by column, then by
// row) give the (row, col) order; duplicates are summed in insertion order.
namespace {
__global__ void triplet_bounds_kernel(const uint32_t* __restrict__ row, const uint32_t* __restrict__ col,
                                      uint64_t n, uint32_t rows, uint32_t cols,
                                      unsigned long long* __restrict__ bad) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n && (row[i] >= rows || col[i] >= cols)) atomicAdd(bad, 1ull);
}
}  // namespace

int triplets_to_csr_launch(sprs_b200_ctx* ctx, uint64_t rows, uint64_t cols, uint64_t n,
                           const uint32_t* d_row, const uint32_t* d_col, const double* d_val,
                           sprs_b200_csmat* t, cudaStream_t s) {
    if (n >= 0xffffffffull || rows > 0xffffffffull || cols > 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE, "from_triplets: needs nnz, rows, cols < 2^32");
    if (n) {  // the reference panics on an out-of-range triplet (TriMatBase::add_triplet asserts);
              // here it would be an out-of-bounds device write in the counting pass
        unsigned long long* d_bad = nullptr;
        unsigned long long h_bad = 0;
        SPRS_CUDA(ctx, cudaMalloc((void**)&d_bad, 8));
        cudaMemsetAsync(d_bad, 0, 8, s);
        triplet_bounds_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_row, d_col, n, (uint32_t)rows,
                                                                          (uint32_t)cols, d_bad);
        ctx->launches += 1;
        cudaMemcpyAsync(&h_bad, d_bad, 8, cudaMemcpyDeviceToHost, s);
        const cudaError_t e = cudaStreamSynchronize(s);
        cudaFree(d_bad);
        if (e != cudaSuccess) SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "from_triplets: %s", cudaGetErrorString(e));
        if (h_bad)
            SPRS_FAIL(ctx, SPRS_B200_ERR_STRUCTURE, "from_triplets: %llu triplet(s) outside %llu x %llu",
                      h_bad, (unsigned long long)rows, (unsigned long long)cols);
    }
    t->ctx = ctx;
    t->storage = SPRS_B200_CSR;
    t->rows = rows;
    t->cols = cols;
    t->outer = rows;
    t->inner = cols;
    t->indptr_bytes = 4;
    t->owns = true;
    t->nnz = 0;
    SPRS_CUDA(ctx, cudaMalloc(&t->d_indptr, (rows + 1) * sizeof(uint32_t) + 16));
    uint32_t *counts = nullptr, *row_s = nullptr, *col_s = nullptr, *flag = nullptr;
    uint64_t *ip64 = nullptr, *uidx = nullptr;
    SortBuffers sb;
    int st = SPRS_B200_OK;
    do {
        if (cudaMalloc((void**)&counts, (rows + 1) * 4) != cudaSuccess ||
            cudaMalloc((void**)&ip64, (rows + 1) * 8) != cudaSuccess) {
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        cudaMemsetAsync(counts, 0, (rows + 1) * 4, s);
        uint64_t n_unique = 0;
        if (n) {
            if (cudaMalloc((void**)&row_s, n * 4) != cudaSuccess ||
                cudaMalloc((void**)&col_s, n * 4) != cudaSuccess ||
                cudaMalloc((void**)&flag, n * 4) != cudaSuccess ||
                cudaMalloc((void**)&uidx, (n + 1) * 8) != cudaSuccess ||
                sb.alloc(n) != SPRS_B200_OK) {
                st = SPRS_B200_ERR_CUDA;
                break;
            }
            const uint32_t *k1 = nullptr, *p1 = nullptr, *k2 = nullptr, *p2 = nullptr;
            if ((st = stable_sort_pairs(ctx, sb, d_col, nullptr, n, bits_for(cols), s, &k1, &p1)) !=
                SPRS_B200_OK)
                break;
            gather_u32_kernel<<<grid_for(n), 256, 0, s>>>(d_row, p1, n, row_s);  // row in col order
            if ((st = stable_sort_pairs(ctx, sb, row_s, p1, n, bits_for(rows), s, &k2, &p2)) !=
                SPRS_B200_OK)
                break;
            gather_u32_kernel<<<grid_for(n), 256, 0, s>>>(d_col, p2, n, col_s);
            head_flags_kernel<<<grid_for(n), 256, 0, s>>>(k2, col_s, n, flag);
            ctx->launches += 3;
            if ((st = device_exclusive_scan<uint32_t, uint64_t>(ctx, flag, n, uidx, s)) != SPRS_B200_OK)
                break;
            if (cudaMemcpyAsync(&n_unique, uidx + n, 8, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
                cudaStreamSynchronize(s) != cudaSuccess) {
                st = SPRS_B200_ERR_CUDA;
                break;
            }
            if (cudaMalloc((void**)&t->d_indices, n_unique * 4 + 16) != cudaSuccess ||
                cudaMalloc((void**)&t->d_data, n_unique * 8 + 16) != cudaSuccess) {
                st = SPRS_B200_ERR_CUDA;
                break;
            }
            compress_runs_kernel<<<grid_for(n), 256, 0, s>>>(k2, col_s, p2, flag, uidx, d_val, n,
                                                            t->d_indices, t->d_data, counts);
            ctx->launches += 1;
        } else {
            if (cudaMalloc((void**)&t->d_indices, 16) != cudaSuccess ||
                cudaMalloc((void**)&t->d_data, 16) != cudaSuccess) {
                st = SPRS_B200_ERR_CUDA;
                break;
            }
        }
        t->nnz = n_unique;
        if ((st = device_exclusive_scan<uint32_t, uint64_t>(ctx, counts, rows, ip64, s)) != SPRS_B200_OK)
            break;
        narrow_kernel<uint64_t, uint32_t><<<grid_for(rows + 1), 256, 0, s>>>(
            ip64, (uint32_t*)t->d_indptr, rows + 1);
        ctx->launches += 1;
    } while (0);
    cudaError_t e = cudaStreamSynchronize(s);
    if (st == SPRS_B200_OK && e == cudaSuccess) e = cudaGetLastError();
    if (st == SPRS_B200_OK && e != cudaSuccess) st = SPRS_B200_ERR_CUDA;
    if (st == SPRS_B200_ERR_CUDA) sprs_b200_set_error(ctx, "from_triplets: CUDA allocation or kernel failed");
    if (counts) cudaFree(counts);
    if (ip64) cudaFree(ip64);
    if (row_s) cudaFree(row_s);
    if (col_s) cudaFree(col_s);
    if (flag) cudaFree(flag);
    if (uidx) cudaFree(uidx);
    sb.release();
    return st;
}

// ---- the dense boundary of a sparse matrix: to_dense / assign_to_dense
// (to_dense.rs:12-30, csmat.rs:1127-1134), csr_from_dense / csc_from_dense (csmat.rs:502-549)
// and the sparse (+) dense binops add_dense_mat_same_ordering / mul_dense_mat_same_ordering
// through csmat_binop_dense_raw (binop.rs:273-433).
//
// Design (DESIGN.md 4.11).  A dense operand is seen in the sparse matrix's outer-major order:
// rows of a CSR matrix, columns of a CSC one, with signed 64-bit element strides (so, si) along
// the outer and inner dimension, so any ndarray view (negative, zero or non-unit strides) works.
//   * MERGE (to_dense, ADD, MUL): the outer x inner positions are one flat run cut into warp
//     tiles of DENSE_TILE consecutive positions.  A tile finds its first stored entry by a binary
//     search of its first row's indices, then walks its positions 32 at a time: the warp keeps a
//     window of 32 stored entries in registers (one coalesced load of indices and values), every
//     entry of the window that falls on the 32 positions sets its bit in a warp OR, and each
//     position lane takes its value from the window lane by shuffle.  Every out element is
//     written exactly once, from the rhs element of the same lane read once just before, so out
//     may be rhs itself (in-place D <- alpha*A + beta*D).  to_dense reads no rhs.
//   * SCATTER (assign_to_dense): tiles of stored entries; positions without an entry are never
//     touched.  O(nnz + outer).
//   * FROM_DENSE: a COUNT pass evaluates |x| > eps per tile, a 64-bit scan (scan.cuh) turns the
//     tile counts into offsets, and a FILL pass writes indices, data and indptr[o+1] of every
//     outer dimension that ends in the tile (empty ones included).  No atomics, no look-back.
//   Values are copied as bits (NaN payloads, -0.0) except in ADD / MUL, which are the reference's
//   closures in IEEE operations: (alpha*x) + (beta*y) and (alpha*x)*y, x = +0.0 where A has no
//   entry.
namespace {

constexpr uint64_t DENSE_TILE = 4096;       // positions per warp tile (merge, from_dense)
constexpr int DENSE_UNROLL = 4;             // 32-position chunks whose rhs loads are in flight
constexpr uint64_t SCATTER_TILE = 256;      // stored entries per warp tile (assign_to_dense)
constexpr uint32_t NO_INDEX = 0xffffffffu;  // inner indices are < 2^32 - 1
constexpr unsigned FULL = 0xffffffffu;

enum { DOP_COPY = 0, DOP_ADD = 1, DOP_MUL = 2 };

// outer-major view of a dense operand: element (o, i) at p[o * so + i * si]
struct DView {
    double* p;
    int64_t so, si;
};

template <typename P>
struct Sparse {
    const P* ip;
    const uint32_t* idx;
    const double* val;
    uint64_t outer, inner;
};

__device__ __forceinline__ int64_t at(const DView& v, uint64_t o, uint64_t i) {
    return (int64_t)o * v.so + (int64_t)i * v.si;
}

// first k in [lo, hi) with idx[k] >= key
__device__ __forceinline__ uint64_t lower_bound_idx(const uint32_t* idx, uint64_t lo, uint64_t hi,
                                                    uint64_t key) {
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if ((uint64_t)idx[mid] < key)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

template <int OP>
__device__ __forceinline__ double dense_op(double x, double y, double alpha, double beta) {
    if (OP == DOP_ADD) return __dadd_rn(__dmul_rn(alpha, x), __dmul_rn(beta, y));
    if (OP == DOP_MUL) return __dmul_rn(__dmul_rn(alpha, x), y);
    return x;
}

// to_dense (OP = COPY: out = A, +0.0 elsewhere) and csmat_binop_dense_raw with the ADD / MUL
// closures.  One warp per tile of DENSE_TILE positions; every loop below is warp-uniform.
template <int OP, typename P>
__global__ void __launch_bounds__(256)
    dense_merge_kernel(Sparse<P> a, uint64_t n_tiles, DView rhs, DView out, double alpha,
                       double beta) {
    const uint64_t t = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (t >= n_tiles) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t total = a.outer * a.inner;
    const uint64_t p0 = t * DENSE_TILE;
    const uint64_t p1 = p0 + DENSE_TILE < total ? p0 + DENSE_TILE : total;
    for (uint64_t o = p0 / a.inner; o < a.outer && o * a.inner < p1; ++o) {
        const uint64_t row0 = o * a.inner;
        const uint64_t i0 = p0 > row0 ? p0 - row0 : 0;
        const uint64_t i1 = p1 - row0 < a.inner ? p1 - row0 : a.inner;
        const uint64_t kend = a.ip[o + 1];
        uint64_t k = i0 ? lower_bound_idx(a.idx, a.ip[o], kend, i0) : (uint64_t)a.ip[o];
        // the window: stored entries wk .. wk+31 of this row (NO_INDEX past its end)
        uint64_t wk = k;
        uint32_t widx = wk + lane < kend ? a.idx[wk + lane] : NO_INDEX;
        double wval = wk + lane < kend ? a.val[wk + lane] : 0.0;
        for (uint64_t base = i0; base < i1; base += 32 * DENSE_UNROLL) {
            double d[DENSE_UNROLL];
#pragma unroll
            for (int u = 0; u < DENSE_UNROLL; ++u) {
                const uint64_t pos = base + u * 32 + lane;
                d[u] = OP != DOP_COPY && pos < i1 ? rhs.p[at(rhs, o, pos)] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < DENSE_UNROLL; ++u) {
                const uint64_t cbase = base + u * 32;
                if (cbase >= i1) break;
                bool has = false;
                double x = 0.0;
                for (;;) {
                    const uint32_t off = (uint32_t)(k - wk);
                    const bool in = lane >= off && (uint64_t)widx < cbase + 32;
                    const uint32_t hits =
                        __reduce_or_sync(FULL, in ? 1u << (uint32_t)(widx - cbase) : 0u);
                    const bool mine = (hits >> lane) & 1u;
                    const uint32_t src = off + __popc(hits & ((1u << lane) - 1u));
                    const double v = __shfl_sync(FULL, wval, mine ? src : 0);
                    if (mine) {
                        has = true;
                        x = v;
                    }
                    k += __popc(hits);
                    if (k - wk < 32 || k >= kend) break;
                    wk = k;  // window used up: the next 32 entries, which may still fall here
                    widx = wk + lane < kend ? a.idx[wk + lane] : NO_INDEX;
                    wval = wk + lane < kend ? a.val[wk + lane] : 0.0;
                }
                const uint64_t pos = cbase + lane;
                if (pos < i1)
                    out.p[at(out, o, pos)] = dense_op<OP>(has ? x : 0.0, d[u], alpha, beta);
            }
        }
    }
}

// assign_to_dense: out(o, idx[k]) = val[k] for every stored entry, nothing else touched.  One warp
// per SCATTER_TILE entries; each lane finds the outer dimension of its entries by walking indptr
// forward from the tile's first one.
template <typename P>
__global__ void __launch_bounds__(256)
    dense_scatter_kernel(Sparse<P> a, uint64_t nnz, uint64_t n_tiles, DView out) {
    const uint64_t t = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (t >= n_tiles) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t k0 = t * SCATTER_TILE;
    uint64_t lo = 0, hi = a.outer;  // the largest o with ip[o] <= k0
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo + 1) / 2;
        if ((uint64_t)a.ip[mid] <= k0)
            lo = mid;
        else
            hi = mid - 1;
    }
    uint64_t o = lo;
    for (uint64_t k = k0 + lane; k < k0 + SCATTER_TILE && k < nnz; k += 32) {
        while ((uint64_t)a.ip[o + 1] <= k) ++o;
        out.p[at(out, o, a.idx[k])] = a.val[k];
    }
}

// from_dense, both passes: the kept test |x| > eps (NaN never kept), COUNT stores the tile's
// count, FILL its entries at the tile's offset and indptr[o+1] of every outer dimension ending here.
template <bool FILL, typename PC>
__global__ void __launch_bounds__(256)
    from_dense_kernel(DView m, uint64_t outer, uint64_t inner, uint64_t n_tiles, double eps,
                      uint32_t* __restrict__ tile_cnt, const uint64_t* __restrict__ tile_off,
                      PC* __restrict__ ipC, uint32_t* __restrict__ iC, double* __restrict__ vC) {
    const uint64_t t = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (t >= n_tiles) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t total = outer * inner;
    const uint64_t p0 = t * DENSE_TILE;
    const uint64_t p1 = p0 + DENSE_TILE < total ? p0 + DENSE_TILE : total;
    uint64_t pos_out = FILL ? tile_off[t] : 0;
    if (FILL && t == 0 && lane == 0) ipC[0] = 0;
    for (uint64_t o = p0 / inner; o < outer && o * inner < p1; ++o) {
        const uint64_t row0 = o * inner;
        const uint64_t i0 = p0 > row0 ? p0 - row0 : 0;
        const uint64_t i1 = p1 - row0 < inner ? p1 - row0 : inner;
        for (uint64_t base = i0; base < i1; base += 32 * DENSE_UNROLL) {
            double x[DENSE_UNROLL];
#pragma unroll
            for (int u = 0; u < DENSE_UNROLL; ++u) {
                const uint64_t pos = base + u * 32 + lane;
                x[u] = pos < i1 ? m.p[at(m, o, pos)] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < DENSE_UNROLL; ++u) {
                const uint64_t pos = base + u * 32 + lane;
                const bool keep = pos < i1 && fabs(x[u]) > eps;
                const uint32_t mask = __ballot_sync(FULL, keep);
                if (FILL && keep) {
                    const uint64_t q = pos_out + __popc(mask & ((1u << lane) - 1u));
                    iC[q] = (uint32_t)pos;
                    vC[q] = x[u];
                }
                pos_out += __popc(mask);
            }
        }
        if (FILL && i1 == inner && lane == 0) ipC[o + 1] = (PC)pos_out;
    }
    if (!FILL && lane == 0) tile_cnt[t] = (uint32_t)pos_out;
}

unsigned warps_grid(uint64_t n_warps) { return (unsigned)((n_warps + 7) / 8); }

// outer-major view of a row-major-strided (rs, cs) operand for a matrix of this storage
DView outer_major(int storage, double* p, int64_t rs, int64_t cs) {
    return storage == SPRS_B200_CSR ? DView{p, rs, cs} : DView{p, cs, rs};
}

template <typename P>
Sparse<P> sparse_of(const sprs_b200_csmat* m) {
    return Sparse<P>{(const P*)m->d_indptr, m->d_indices, m->d_data, m->outer, m->inner};
}

int merge_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, int dop, DView rhs, DView out,
                 double alpha, double beta, cudaStream_t s) {
    const uint64_t total = m->outer * m->inner;
    if (total == 0) return SPRS_B200_OK;
    const uint64_t n_tiles = (total + DENSE_TILE - 1) / DENSE_TILE;
    const unsigned g = warps_grid(n_tiles);
#define SPRS_DENSE_MERGE(OP, P) \
    dense_merge_kernel<OP, P><<<g, 256, 0, s>>>(sparse_of<P>(m), n_tiles, rhs, out, alpha, beta)
    const bool p64 = m->indptr_bytes == 8;
    if (dop == DOP_COPY) {
        if (p64) SPRS_DENSE_MERGE(DOP_COPY, uint64_t); else SPRS_DENSE_MERGE(DOP_COPY, uint32_t);
    } else if (dop == DOP_ADD) {
        if (p64) SPRS_DENSE_MERGE(DOP_ADD, uint64_t); else SPRS_DENSE_MERGE(DOP_ADD, uint32_t);
    } else {
        if (p64) SPRS_DENSE_MERGE(DOP_MUL, uint64_t); else SPRS_DENSE_MERGE(DOP_MUL, uint32_t);
    }
#undef SPRS_DENSE_MERGE
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

int scatter_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, DView out, cudaStream_t s) {
    if (m->nnz == 0) return SPRS_B200_OK;
    const uint64_t n_tiles = (m->nnz + SCATTER_TILE - 1) / SCATTER_TILE;
    if (m->indptr_bytes == 8)
        dense_scatter_kernel<uint64_t><<<warps_grid(n_tiles), 256, 0, s>>>(sparse_of<uint64_t>(m),
                                                                           m->nnz, n_tiles, out);
    else
        dense_scatter_kernel<uint32_t><<<warps_grid(n_tiles), 256, 0, s>>>(sparse_of<uint32_t>(m),
                                                                           m->nnz, n_tiles, out);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

// both passes of from_dense into a new device mirror (blocking on s)
int from_dense_run(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols, DView m,
                   double epsilon, cudaStream_t s, sprs_b200_csmat** out) {
    const double eps = epsilon > 0.0 ? epsilon : 0.0;  // csmat.rs:506-510: NaN and <= 0 -> 0
    const uint64_t outer = storage == SPRS_B200_CSR ? rows : cols;
    const uint64_t inner = storage == SPRS_B200_CSR ? cols : rows;
    const uint64_t total = outer * inner;
    const uint64_t n_tiles = (total + DENSE_TILE - 1) / DENSE_TILE;
    uint32_t* cnt = nullptr;
    uint64_t* off = nullptr;
    sprs_b200_csmat* c = nullptr;
    int st = SPRS_B200_OK;
    do {
        uint64_t nnz = 0;
        if (n_tiles) {
            if (cudaMallocAsync((void**)&cnt, n_tiles * 4, s) != cudaSuccess ||
                cudaMallocAsync((void**)&off, (n_tiles + 1) * 8, s) != cudaSuccess) {
                cudaGetLastError();
                sprs_b200_set_error(ctx, "from_dense: cudaMallocAsync of the tile counts failed");
                st = SPRS_B200_ERR_CUDA;
                break;
            }
            from_dense_kernel<false, uint32_t><<<warps_grid(n_tiles), 256, 0, s>>>(
                m, outer, inner, n_tiles, eps, cnt, nullptr, nullptr, nullptr, nullptr);
            ctx->launches += 1;
            if ((st = device_exclusive_scan<uint32_t, uint64_t>(ctx, cnt, n_tiles, off, s)) !=
                SPRS_B200_OK)
                break;
            if (cudaMemcpyAsync(&nnz, off + n_tiles, 8, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
                cudaStreamSynchronize(s) != cudaSuccess) {
                sprs_b200_set_error(ctx, "from_dense: count pass failed");
                st = SPRS_B200_ERR_CUDA;
                break;
            }
        }
        c = new_result(ctx, storage, rows, cols, nnz,
                       (nnz >= 0xffffffffull || force_indptr64()) ? 8 : 4);
        if ((st = alloc_result(ctx, c, s)) != SPRS_B200_OK) break;
        if (n_tiles == 0) {  // no position: indptr is all zeros
            if (cudaMemsetAsync(c->d_indptr, 0, (outer + 1) * (size_t)c->indptr_bytes, s) !=
                cudaSuccess) {
                sprs_b200_set_error(ctx, "from_dense: memset failed");
                st = SPRS_B200_ERR_CUDA;
                break;
            }
        } else if (c->indptr_bytes == 4) {
            from_dense_kernel<true, uint32_t><<<warps_grid(n_tiles), 256, 0, s>>>(
                m, outer, inner, n_tiles, eps, nullptr, off, (uint32_t*)c->d_indptr, c->d_indices,
                c->d_data);
        } else {
            from_dense_kernel<true, uint64_t><<<warps_grid(n_tiles), 256, 0, s>>>(
                m, outer, inner, n_tiles, eps, nullptr, off, (uint64_t*)c->d_indptr, c->d_indices,
                c->d_data);
        }
        ctx->launches += n_tiles ? 1 : 0;
        if (cudaGetLastError() != cudaSuccess) {
            sprs_b200_set_error(ctx, "from_dense: launch failed");
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        st = finish_result(ctx, c, s, "from_dense");
    } while (0);
    if (cnt) cudaFreeAsync(cnt, s);
    if (off) cudaFreeAsync(off, s);
    if (st != SPRS_B200_OK) {
        sprs_b200_csmat_free(c);
        return st;
    }
    *out = c;
    return SPRS_B200_OK;
}

// ---- host-buffer plumbing: a strided host view <-> a contiguous outer-major device copy,
// through the pinned staging buffer (O(size) copies, no arithmetic)
void pack(const double* v, int64_t so, int64_t si, uint64_t outer, uint64_t inner, double* dst) {
    for (uint64_t o = 0; o < outer; ++o)
        for (uint64_t i = 0; i < inner; ++i) dst[o * inner + i] = v[(int64_t)o * so + (int64_t)i * si];
}

void unpack(const double* src, uint64_t outer, uint64_t inner, double* v, int64_t so, int64_t si) {
    for (uint64_t o = 0; o < outer; ++o)
        for (uint64_t i = 0; i < inner; ++i) v[(int64_t)o * so + (int64_t)i * si] = src[o * inner + i];
}

// the device scratch copy (slot `slot`) of a host view, packed outer-major; upload=false only
// reserves it
int stage_in(sprs_b200_ctx* ctx, int slot, const double* v, int64_t so, int64_t si, uint64_t outer,
             uint64_t inner, bool upload, double** d) {
    const size_t n = (size_t)(outer * inner);
    SPRS_TRY(ctx_scratch(ctx, slot, n * 8, (void**)d));
    if (!upload || n == 0) return SPRS_B200_OK;
    void* hs = nullptr;
    SPRS_TRY(ctx_stage(ctx, n * 8, &hs));
    pack(v, so, si, outer, inner, (double*)hs);
    SPRS_CUDA(ctx, cudaMemcpyAsync(*d, hs, n * 8, cudaMemcpyHostToDevice, ctx->stream));
    SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the staging buffer is reused
    return SPRS_B200_OK;
}

int stage_out(sprs_b200_ctx* ctx, const double* d, uint64_t outer, uint64_t inner, double* v,
              int64_t so, int64_t si) {
    const size_t n = (size_t)(outer * inner);
    if (n == 0) return SPRS_B200_OK;
    void* hs = nullptr;
    SPRS_TRY(ctx_stage(ctx, n * 8, &hs));
    SPRS_CUDA(ctx, cudaMemcpyAsync(hs, d, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    unpack((const double*)hs, outer, inner, v, so, si);
    return SPRS_B200_OK;
}

// csmat_binop_dense_raw's checks (binop.rs:400-418), then the op code: the reference has no
// dense subtraction.  fastest_axis (sparse.rs:400-406): Axis(0) iff strides[1] > strides[0].
int binop_dense_check(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs, int op, uint64_t rhs_rows,
                      uint64_t rhs_cols, int64_t rhs_rs, int64_t rhs_cs, uint64_t out_rows,
                      uint64_t out_cols, int64_t out_rs, int64_t out_cs, int* dop) {
    if (lhs->cols != rhs_cols || lhs->cols != out_cols || lhs->rows != rhs_rows ||
        lhs->rows != out_rows)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    const bool rhs_f = rhs_cs > rhs_rs, out_f = out_cs > out_rs;
    const bool csr = lhs->storage == SPRS_B200_CSR;
    if (!((csr && !rhs_f && !out_f) || (!csr && rhs_f && out_f)))
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch");
    if (op == SPRS_B200_BINOP_ADD)
        *dop = DOP_ADD;
    else if (op == SPRS_B200_BINOP_MUL)
        *dop = DOP_MUL;
    else
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "binop_dense: op %d (only ADD and MUL)", op);
    return SPRS_B200_OK;
}

int from_dense_check(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols) {
    if (storage != SPRS_B200_CSR && storage != SPRS_B200_CSC)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "from_dense: bad storage %d", storage);
    if (rows > 0xffffffffull || cols > 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE,
                  "Index type is not large enough: device mirrors use u32 indices");
    return SPRS_B200_OK;
}

}  // namespace

extern "C" {

int sprs_b200_csmat_to_dense_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, double* d_out,
                                 uint64_t ld, void* stream) {
    if (!ctx || !m || (!d_out && m->rows && m->cols)) return SPRS_B200_ERR_ARGUMENT;
    if (ld < m->cols) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch: ld < cols");
    const DView out = outer_major(m->storage, d_out, (int64_t)ld, 1);
    return merge_launch(ctx, m, DOP_COPY, DView{nullptr, 0, 0}, out, 0.0, 0.0,
                        pick_stream(ctx, stream));
}

int sprs_b200_csmat_to_dense(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, double* out,
                             uint64_t ld) {
    if (!ctx || !m || (!out && m->rows && m->cols)) return SPRS_B200_ERR_ARGUMENT;
    if (ld < m->cols) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch: ld < cols");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    double* d = nullptr;
    SPRS_TRY(stage_in(ctx, 1, nullptr, 0, 0, m->outer, m->inner, false, &d));
    SPRS_TRY(merge_launch(ctx, m, DOP_COPY, DView{nullptr, 0, 0}, DView{d, (int64_t)m->inner, 1},
                          0.0, 0.0, ctx->stream));
    const DView o = outer_major(m->storage, out, (int64_t)ld, 1);
    return stage_out(ctx, d, m->outer, m->inner, out, o.so, o.si);
}

int sprs_b200_assign_to_dense_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, double* d_out,
                                  uint64_t rows, uint64_t cols, int64_t rs, int64_t cs,
                                  void* stream) {
    if (!ctx || !m) return SPRS_B200_ERR_ARGUMENT;
    // to_dense.rs:20-21: cols first, then rows
    if (m->cols != cols || m->rows != rows) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (!d_out && m->nnz) return SPRS_B200_ERR_ARGUMENT;
    return scatter_launch(ctx, m, outer_major(m->storage, d_out, rs, cs), pick_stream(ctx, stream));
}

int sprs_b200_assign_to_dense(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, double* out,
                              uint64_t rows, uint64_t cols, int64_t rs, int64_t cs) {
    if (!ctx || !m) return SPRS_B200_ERR_ARGUMENT;
    if (m->cols != cols || m->rows != rows) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (m->nnz == 0) return SPRS_B200_OK;
    if (!out) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    const DView o = outer_major(m->storage, out, rs, cs);
    double* d = nullptr;
    SPRS_TRY(stage_in(ctx, 1, out, o.so, o.si, m->outer, m->inner, true, &d));
    SPRS_TRY(scatter_launch(ctx, m, DView{d, (int64_t)m->inner, 1}, ctx->stream));
    return stage_out(ctx, d, m->outer, m->inner, out, o.so, o.si);
}

int sprs_b200_csmat_from_dense_dev(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                                   const double* d_m, int64_t rs, int64_t cs, double epsilon,
                                   sprs_b200_csmat** out) {
    if (!ctx || !out || (!d_m && rows && cols)) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_TRY(from_dense_check(ctx, storage, rows, cols));
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    return from_dense_run(ctx, storage, rows, cols, outer_major(storage, (double*)d_m, rs, cs),
                          epsilon, ctx->stream, out);
}

int sprs_b200_csmat_from_dense(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                               const double* m, int64_t rs, int64_t cs, double epsilon,
                               sprs_b200_csmat** out) {
    if (!ctx || !out || (!m && rows && cols)) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_TRY(from_dense_check(ctx, storage, rows, cols));
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    const DView v = outer_major(storage, (double*)m, rs, cs);
    const uint64_t outer = storage == SPRS_B200_CSR ? rows : cols;
    const uint64_t inner = storage == SPRS_B200_CSR ? cols : rows;
    double* d = nullptr;
    SPRS_TRY(stage_in(ctx, 1, m, v.so, v.si, outer, inner, true, &d));
    return from_dense_run(ctx, storage, rows, cols, DView{d, (int64_t)inner, 1}, epsilon,
                          ctx->stream, out);
}

int sprs_b200_csmat_binop_dense_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs, int op,
                                    double alpha, double beta, const double* d_rhs,
                                    uint64_t rhs_rows, uint64_t rhs_cols, int64_t rhs_rs,
                                    int64_t rhs_cs, double* d_out, uint64_t out_rows,
                                    uint64_t out_cols, int64_t out_rs, int64_t out_cs,
                                    void* stream) {
    if (!ctx || !lhs) return SPRS_B200_ERR_ARGUMENT;
    int dop = 0;
    SPRS_TRY(binop_dense_check(ctx, lhs, op, rhs_rows, rhs_cols, rhs_rs, rhs_cs, out_rows,
                               out_cols, out_rs, out_cs, &dop));
    if ((!d_rhs || !d_out) && lhs->rows && lhs->cols) return SPRS_B200_ERR_ARGUMENT;
    return merge_launch(ctx, lhs, dop, outer_major(lhs->storage, (double*)d_rhs, rhs_rs, rhs_cs),
                        outer_major(lhs->storage, d_out, out_rs, out_cs), alpha, beta,
                        pick_stream(ctx, stream));
}

int sprs_b200_csmat_binop_dense(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs, int op,
                                double alpha, double beta, const double* rhs, uint64_t rhs_rows,
                                uint64_t rhs_cols, int64_t rhs_rs, int64_t rhs_cs, double* out,
                                uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                int64_t out_cs) {
    if (!ctx || !lhs) return SPRS_B200_ERR_ARGUMENT;
    int dop = 0;
    SPRS_TRY(binop_dense_check(ctx, lhs, op, rhs_rows, rhs_cols, rhs_rs, rhs_cs, out_rows,
                               out_cols, out_rs, out_cs, &dop));
    if (lhs->rows == 0 || lhs->cols == 0) return SPRS_B200_OK;
    if (!rhs || !out) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    const DView r = outer_major(lhs->storage, (double*)rhs, rhs_rs, rhs_cs);
    const DView o = outer_major(lhs->storage, out, out_rs, out_cs);
    double *d_rhs = nullptr, *d_out = nullptr;
    SPRS_TRY(stage_in(ctx, 1, rhs, r.so, r.si, lhs->outer, lhs->inner, true, &d_rhs));
    SPRS_TRY(stage_in(ctx, 2, nullptr, 0, 0, lhs->outer, lhs->inner, false, &d_out));
    const int64_t ld = (int64_t)lhs->inner;
    SPRS_TRY(merge_launch(ctx, lhs, dop, DView{d_rhs, ld, 1}, DView{d_out, ld, 1}, alpha, beta,
                          ctx->stream));
    return stage_out(ctx, d_out, lhs->outer, lhs->inner, out, o.so, o.si);
}

}  // extern "C"
