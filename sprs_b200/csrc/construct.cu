// construct.cu -- sparse matrix construction for sm_90a: block concatenation (bmat, vstack,
// hstack) and the Kronecker product.
//
// Replaces sprs::bmat / vstack / hstack (sprs/src/sparse/construct.rs) and
// sprs::kronecker_product (sprs/src/sparse/kronecker.rs).  Both are pure output streams, so the
// result is bit-identical to the reference by construction: stacking copies every value as a
// 64-bit word (NaN payloads and -0.0 survive), the Kronecker product rounds one IEEE multiply
// per output entry (__dmul_rn, no FMA) and drops nothing.
//
// Design (DESIGN.md 4.10).
//   * ONE concatenation kernel.  Blocks are CSR (CSC blocks arrive as their cached device
//     conversion, csmat_csr_view).  The block table -- each present block's arrays, indptr
//     width and column offset, each block row's first output row, first output non-zero and
//     first block -- lives in device memory, so grids of any size work.
//       INDPTR  one thread per output row R = R_I + r of block row I:
//               ipC[R] = base_I + sum_J (ip_IJ[r] - ip_IJ[0]) over the present blocks of row I.
//       FILL    a warp owns CONSTRUCT_TILE consecutive OUTPUT entries (not rows): a binary
//               search of ipC gives the row of its first entry, then it walks the (row, block)
//               segments in output order and copies the part of each inside its range with
//               coalesced 32-lane loads and stores, adding the block's column offset to each
//               index.  A hub row is spread over as many warps as it has tiles; a run of empty
//               rows is jumped over by another binary search of ipC.
//   * ONE Kronecker kernel, in the outer / inner view of a's storage (b already converted):
//       INDPTR  closed form, no scan: ipC[ia*outer(b) + ib] = ipA[ia]*nnz(b) + lenA(ia)*ipB[ib].
//       FILL    tiled by output position like the concatenation.  Output row (ia, ib) lists,
//               for each entry p of a's vector ia, each entry q of b's vector ib.  A row of 32
//               entries or more: a lane finds its first (p, q) with one division and then steps
//               32 entries at a time incrementally.  A shorter row: the warp takes the next 32
//               rows at once (one lane reads each row's indptr entries, so the reads overlap)
//               and each output entry finds its row by a 5-step shuffle search over the lanes'
//               row starts.  Index ja*inner(b) + jb in 64 bits, value __dmul_rn(va, vb).
//   * Results come from new_result / alloc_result / finish_result (binop.cu): stream-ordered
//     pool arrays, 64-bit indptr exactly when nnz >= 2^32 - 1 (or SPRS_B200_FORCE_INDPTR64),
//     the SpMV partition built.  No atomics, no waits between CTAs: deterministic.
//   * Every contract check runs on the host before any device work.

#include "common.cuh"

#include <algorithm>
#include <vector>

namespace {

constexpr uint64_t CONSTRUCT_TILE = 2048;  // output entries per warp tile (both fill kernels)
constexpr uint64_t U32_DIM = 0xffffffffull;  // device mirrors index dimensions with u32

struct Block {
    const void* ip;              // outer + 1 entries, u32 or u64 (ip64)
    const uint32_t* idx;
    const unsigned long long* val;  // values moved as 64-bit words
    uint64_t col_off;            // columns of the blocks to its left in its block row
    uint32_t ip64;
    uint32_t pad;
};

struct Table {
    const Block* blk;       // present blocks, block row by block row, left to right
    const uint64_t* row0;   // n_brow + 1: first output row of block row I
    const uint64_t* base;   // n_brow + 1: first output non-zero of block row I
    const uint64_t* first;  // n_brow + 1: first block of block row I in blk
    uint64_t n_brow;
};

__device__ __forceinline__ uint64_t ld_ip(const Block& b, uint64_t r) {
    return b.ip64 ? __ldg((const unsigned long long*)b.ip + r) : __ldg((const uint32_t*)b.ip + r);
}

// the largest R in [lo, hi] with ip[R] <= pos (ip[lo] <= pos)
template <typename P>
__device__ __forceinline__ uint64_t last_le(const P* ip, uint64_t lo, uint64_t hi, uint64_t pos) {
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo + 1) / 2;
        if ((uint64_t)ip[mid] <= pos)
            lo = mid;
        else
            hi = mid - 1;
    }
    return lo;
}

// the row that holds output entry pos (pos < nnz), searching from row lo: the next row when it
// is not empty, else a binary search over the run of empty rows
template <typename P>
__device__ __forceinline__ uint64_t row_of(const P* ip, uint64_t lo, uint64_t rows, uint64_t pos) {
    if (lo + 1 >= rows || (uint64_t)ip[lo + 1] > pos) return lo;
    return last_le(ip, lo + 1, rows - 1, pos);
}

// the block row of output row R (the last one starting at or before R: skips 0-row block rows)
__device__ __forceinline__ uint64_t brow_of(const Table& t, uint64_t R) {
    uint64_t lo = 0, hi = t.n_brow - 1;
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo + 1) / 2;
        if (t.row0[mid] <= R)
            lo = mid;
        else
            hi = mid - 1;
    }
    return lo;
}

template <typename PC>
__global__ void bmat_indptr_kernel(Table t, uint64_t rows, PC* __restrict__ ipC) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t R = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; R <= rows; R += stride) {
        if (R == rows) {
            ipC[R] = (PC)t.base[t.n_brow];
            continue;
        }
        const uint64_t I = brow_of(t, R);
        const uint64_t r = R - t.row0[I];
        uint64_t acc = t.base[I];
        for (uint64_t j = t.first[I]; j < t.first[I + 1]; ++j) {
            const Block b = t.blk[j];
            acc += ld_ip(b, r) - ld_ip(b, 0);
        }
        ipC[R] = (PC)acc;
    }
}

template <typename PC>
__global__ void __launch_bounds__(256)
    bmat_fill_kernel(Table t, uint64_t rows, uint64_t nnz, uint64_t n_tiles,
                     const PC* __restrict__ ipC, uint32_t* __restrict__ iC,
                     unsigned long long* __restrict__ vC) {
    const uint64_t w = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (w >= n_tiles) return;
    const uint64_t lane = threadIdx.x & 31;
    const uint64_t k0 = w * CONSTRUCT_TILE;
    const uint64_t k1 = k0 + CONSTRUCT_TILE < nnz ? k0 + CONSTRUCT_TILE : nnz;
    uint64_t R = last_le(ipC, 0, rows - 1, k0);
    uint64_t I = brow_of(t, R);
    uint64_t pos = ipC[R];
    for (;;) {
        const uint64_t r = R - t.row0[I];
        for (uint64_t j = t.first[I]; j < t.first[I + 1]; ++j) {
            const Block b = t.blk[j];
            const uint64_t s = ld_ip(b, r), len = ld_ip(b, r + 1) - s;
            if (pos + len > k0) {  // the segment [pos, pos + len) meets [k0, k1)
                const uint64_t lo = pos > k0 ? pos : k0;
                const uint64_t hi = pos + len < k1 ? pos + len : k1;
                const uint32_t off = (uint32_t)b.col_off;
                for (uint64_t q = lo + lane; q < hi; q += 32) {
                    const uint64_t src = s + (q - pos);
                    iC[q] = __ldg(b.idx + src) + off;
                    vC[q] = __ldg(b.val + src);
                }
            }
            pos += len;
            if (pos >= k1) return;
        }
        R = row_of(ipC, R + 1, rows, pos);
        while (t.row0[I + 1] <= R) ++I;
    }
}

struct KronOperands {
    const void* ipA;
    const uint32_t* iA;
    const double* vA;
    const void* ipB;
    const uint32_t* iB;
    const double* vB;
    uint64_t outer_b, inner_b, nnz_b;
    uint32_t a64, b64;
};

__device__ __forceinline__ uint64_t ld_ip(const void* ip, uint32_t ip64, uint64_t r) {
    return ip64 ? __ldg((const unsigned long long*)ip + r) : __ldg((const uint32_t*)ip + r);
}

template <typename PC>
__global__ void kron_indptr_kernel(KronOperands o, uint64_t outer_c, uint64_t nnz_c,
                                   PC* __restrict__ ipC) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t a0 = ld_ip(o.ipA, o.a64, 0), b0 = ld_ip(o.ipB, o.b64, 0);
    for (uint64_t R = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; R <= outer_c; R += stride) {
        if (R == outer_c) {
            ipC[R] = (PC)nnz_c;
            continue;
        }
        const uint64_t ia = R / o.outer_b, ib = R - ia * o.outer_b;
        const uint64_t pa = ld_ip(o.ipA, o.a64, ia);
        const uint64_t la = ld_ip(o.ipA, o.a64, ia + 1) - pa;
        ipC[R] = (PC)((pa - a0) * o.nnz_b + la * (ld_ip(o.ipB, o.b64, ib) - b0));
    }
}

template <typename PC>
__global__ void __launch_bounds__(256)
    kron_fill_kernel(KronOperands o, uint64_t outer_c, uint64_t nnz_c, uint64_t n_tiles,
                     const PC* __restrict__ ipC, uint32_t* __restrict__ iC,
                     double* __restrict__ vC) {
    const uint64_t w = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (w >= n_tiles) return;
    const uint64_t lane = threadIdx.x & 31;
    const uint64_t k0 = w * CONSTRUCT_TILE;
    const uint64_t k1 = k0 + CONSTRUCT_TILE < nnz_c ? k0 + CONSTRUCT_TILE : nnz_c;
    uint64_t R = last_le(ipC, 0, outer_c - 1, k0);
    uint64_t pos = ipC[R];
    for (;;) {
        const uint64_t ia = R / o.outer_b, ib = R - ia * o.outer_b;
        const uint64_t sa = ld_ip(o.ipA, o.a64, ia), la = ld_ip(o.ipA, o.a64, ia + 1) - sa;
        const uint64_t sb = ld_ip(o.ipB, o.b64, ib), lb = ld_ip(o.ipB, o.b64, ib + 1) - sb;
        const uint64_t len = la * lb;  // > 0: row_of only stops on rows that hold pos
        if (len < 32) {
            // a short row: rows R .. R+31 at once, one per lane, so that their indptr reads
            // overlap; each output entry finds its row by a search over the lanes' row starts
            const uint64_t r = R + lane;
            uint64_t rs = nnz_c, re = nnz_c, rsa = 0, rsb = 0, rlb = 1;
            if (r < outer_c) {
                rs = ipC[r];
                re = ipC[r + 1];
                const uint64_t ra = r / o.outer_b, rb = r - ra * o.outer_b;
                rsa = ld_ip(o.ipA, o.a64, ra);
                rsb = ld_ip(o.ipB, o.b64, rb);
                const uint64_t n = ld_ip(o.ipB, o.b64, rb + 1) - rsb;
                rlb = n ? n : 1;  // an empty row of b holds no entry: never searched for
            }
            const uint64_t last = __shfl_sync(0xffffffffu, re, 31);
            const uint64_t hi = last < k1 ? last : k1;
            const uint64_t lo = pos > k0 ? pos : k0;
            for (uint64_t base = lo; base < hi; base += 32) {
                const uint64_t q = base + lane;
                uint32_t j = 0;  // the last lane whose row starts at or before q
                for (uint32_t step = 16; step; step >>= 1) {
                    const uint64_t s = __shfl_sync(0xffffffffu, rs, j + step);
                    if (s <= q) j += step;
                }
                const uint64_t s = __shfl_sync(0xffffffffu, rs, j);
                const uint64_t jsa = __shfl_sync(0xffffffffu, rsa, j);
                const uint64_t jsb = __shfl_sync(0xffffffffu, rsb, j);
                const uint64_t jlb = __shfl_sync(0xffffffffu, rlb, j);
                if (q < hi) {
                    const uint64_t m = q - s;
                    const uint64_t p = (m | jlb) >> 32 ? m / jlb : (uint32_t)m / (uint32_t)jlb;
                    const uint64_t qb = m - p * jlb;
                    const uint64_t ja = __ldg(o.iA + jsa + p), jb = __ldg(o.iB + jsb + qb);
                    iC[q] = (uint32_t)(ja * o.inner_b + jb);
                    vC[q] = __dmul_rn(__ldg(o.vA + jsa + p), __ldg(o.vB + jsb + qb));
                }
            }
            if (hi >= k1) return;
            pos = hi;  // the end of row R + 31
            R = row_of(ipC, R + 32, outer_c, pos);
            continue;
        }
        const uint64_t hi = pos + len < k1 ? pos + len : k1;
        uint64_t q = (pos > k0 ? pos : k0) + lane;
        if (q < hi) {
            const uint64_t m = q - pos;
            uint64_t p = m / lb, qb = m - p * lb;          // once per row ...
            const uint64_t dp = 32 / lb, dq = 32 - dp * lb;  // ... then 32 entries a step
            for (; q < hi; q += 32) {
                const uint64_t ja = __ldg(o.iA + sa + p), jb = __ldg(o.iB + sb + qb);
                iC[q] = (uint32_t)(ja * o.inner_b + jb);
                vC[q] = __dmul_rn(__ldg(o.vA + sa + p), __ldg(o.vB + sb + qb));
                p += dp;
                qb += dq;
                if (qb >= lb) {
                    qb -= lb;
                    ++p;
                }
            }
        }
        pos += len;
        if (pos >= k1) return;
        R = row_of(ipC, R + 1, outer_c, pos);
    }
}

unsigned grid_for(const sprs_b200_ctx* ctx, uint64_t n) {
    return (unsigned)std::max<uint64_t>(
        1, std::min<uint64_t>((n + 255) / 256, (uint64_t)ctx->sm_count * 16));
}

// a pooled result mirror of the given storage and shape
sprs_b200_csmat* construct_result(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                                  uint64_t nnz) {
    sprs_b200_csmat like;
    like.storage = storage;
    like.rows = rows;
    like.cols = cols;
    like.outer = storage == SPRS_B200_CSR ? rows : cols;
    like.inner = storage == SPRS_B200_CSR ? cols : rows;
    return new_result(ctx, &like, nnz, (nnz >= 0xffffffffull || force_indptr64()) ? 8 : 4);
}

bool mul_overflows(uint64_t a, uint64_t b, uint64_t* out) {
    return __builtin_mul_overflow(a, b, out);
}

}  // namespace

extern "C" {

int sprs_b200_csmat_bmat(sprs_b200_ctx* ctx, uint64_t n_block_rows, uint64_t n_block_cols,
                         const sprs_b200_csmat* const* blocks, sprs_b200_csmat** out) {
    if (!ctx || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    // construct.rs bmat: the asserts in its order, then hstack per block row, then vstack
    if (n_block_rows == 0 || n_block_cols == 0)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "Empty stacking list");
    if (!blocks) return SPRS_B200_ERR_ARGUMENT;
    const uint64_t nbr = n_block_rows, nbc = n_block_cols;
    auto at = [&](uint64_t i, uint64_t j) { return blocks[i * nbc + j]; };
    for (uint64_t i = 0; i < nbr; ++i) {
        bool any = false;
        for (uint64_t j = 0; j < nbc && !any; ++j) any = at(i, j) != nullptr;
        if (!any) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "Empty bmat row");
    }
    for (uint64_t j = 0; j < nbc; ++j) {
        bool any = false;
        for (uint64_t i = 0; i < nbr && !any; ++i) any = at(i, j) != nullptr;
        if (!any) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "Empty bmat col");
    }
    std::vector<uint64_t> rows_per_row(nbr, 0), cols_per_col(nbc, 0);
    for (uint64_t i = 0; i < nbr; ++i)
        for (uint64_t j = 0; j < nbc; ++j)
            if (const sprs_b200_csmat* m = at(i, j)) {
                rows_per_row[i] = std::max(rows_per_row[i], m->rows);
                cols_per_col[j] = std::max(cols_per_col[j], m->cols);
            }
    // hstack of block row i: every block (a None is zero(rows_per_row[i], cols_per_col[j])) must
    // have the row's height; its width is the sum of its blocks' widths.  vstack: equal widths.
    uint64_t width0 = 0, rows = 0, nnz = 0;
    for (uint64_t i = 0; i < nbr; ++i) {
        uint64_t width = 0;
        for (uint64_t j = 0; j < nbc; ++j) {
            const sprs_b200_csmat* m = at(i, j);
            if (m && m->rows != rows_per_row[i])
                SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
            width += m ? m->cols : cols_per_col[j];
            if (m) nnz += m->nnz;
        }
        if (i == 0) width0 = width;
        if (width != width0) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
        rows += rows_per_row[i];
        if (width > U32_DIM || rows > U32_DIM)
            SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE,
                      "Index type is not large enough: the result has a dimension >= 2^32 "
                      "(device mirrors use u32 indices)");
    }
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;

    // the block table: CSR form of every present block (CSC ones through their cached conversion)
    std::vector<Block> blk;
    std::vector<uint64_t> row0(nbr + 1), base(nbr + 1), first(nbr + 1);
    for (uint64_t i = 0; i < nbr; ++i) {
        row0[i + 1] = row0[i] + rows_per_row[i];
        base[i + 1] = base[i];
        first[i] = blk.size();
        uint64_t off = 0;
        for (uint64_t j = 0; j < nbc; ++j) {
            const sprs_b200_csmat* m = at(i, j);
            if (!m) {
                off += cols_per_col[j];
                continue;
            }
            const sprs_b200_csmat* c = nullptr;
            SPRS_TRY(csmat_csr_view(ctx, m, &c));
            blk.push_back(Block{c->d_indptr, c->d_indices, (const unsigned long long*)c->d_data,
                                off, c->indptr_bytes == 8 ? 1u : 0u, 0u});
            off += m->cols;
            base[i + 1] += m->nnz;
        }
    }
    first[nbr] = blk.size();

    sprs_b200_csmat* c = construct_result(ctx, SPRS_B200_CSR, rows, width0, nnz);
    void* d_table = nullptr;
    int st = SPRS_B200_OK;
    do {
        if ((st = alloc_result(ctx, c, s)) != SPRS_B200_OK) break;
        const size_t blk_bytes = blk.size() * sizeof(Block), tab_bytes = (nbr + 1) * 8;
        std::vector<unsigned char> host(blk_bytes + 3 * tab_bytes);
        memcpy(host.data(), blk.data(), blk_bytes);
        memcpy(host.data() + blk_bytes, row0.data(), tab_bytes);
        memcpy(host.data() + blk_bytes + tab_bytes, base.data(), tab_bytes);
        memcpy(host.data() + blk_bytes + 2 * tab_bytes, first.data(), tab_bytes);
        if (cudaMallocAsync(&d_table, host.size(), s) != cudaSuccess ||
            cudaMemcpyAsync(d_table, host.data(), host.size(), cudaMemcpyHostToDevice, s) !=
                cudaSuccess) {
            cudaGetLastError();
            sprs_b200_set_error(ctx, "bmat: upload of the block table failed");
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        const unsigned char* d = (const unsigned char*)d_table;
        const Table t{(const Block*)d, (const uint64_t*)(d + blk_bytes),
                      (const uint64_t*)(d + blk_bytes + tab_bytes),
                      (const uint64_t*)(d + blk_bytes + 2 * tab_bytes), nbr};
        const uint64_t n_tiles = (nnz + CONSTRUCT_TILE - 1) / CONSTRUCT_TILE;
        const unsigned fill_grid = (unsigned)((n_tiles + 7) / 8);
        if (c->indptr_bytes == 4) {
            bmat_indptr_kernel<uint32_t><<<grid_for(ctx, rows + 1), 256, 0, s>>>(
                t, rows, (uint32_t*)c->d_indptr);
            if (n_tiles)
                bmat_fill_kernel<uint32_t><<<fill_grid, 256, 0, s>>>(
                    t, rows, nnz, n_tiles, (const uint32_t*)c->d_indptr, c->d_indices,
                    (unsigned long long*)c->d_data);
        } else {
            bmat_indptr_kernel<uint64_t><<<grid_for(ctx, rows + 1), 256, 0, s>>>(
                t, rows, (uint64_t*)c->d_indptr);
            if (n_tiles)
                bmat_fill_kernel<uint64_t><<<fill_grid, 256, 0, s>>>(
                    t, rows, nnz, n_tiles, (const uint64_t*)c->d_indptr, c->d_indices,
                    (unsigned long long*)c->d_data);
        }
        ctx->launches += n_tiles ? 2 : 1;
        if (cudaGetLastError() != cudaSuccess) {
            sprs_b200_set_error(ctx, "bmat: launch failed");
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        st = finish_result(ctx, c, s, "bmat");
    } while (0);
    if (d_table) cudaFreeAsync(d_table, s);
    if (st != SPRS_B200_OK) {
        sprs_b200_csmat_free(c);
        return st;
    }
    *out = c;
    return SPRS_B200_OK;
}

int sprs_b200_csmat_kron(sprs_b200_ctx* ctx, const sprs_b200_csmat* a, const sprs_b200_csmat* b,
                         sprs_b200_csmat** out) {
    if (!ctx || !a || !b || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    uint64_t rows, cols, nnz;
    if (mul_overflows(a->rows, b->rows, &rows) || mul_overflows(a->cols, b->cols, &cols) ||
        mul_overflows(a->nnz, b->nnz, &nnz))
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE, "kron: the result's shape or nnz overflows 64 bits");
    if (rows > U32_DIM || cols > U32_DIM)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE,
                  "Index type is not large enough: the result has a dimension >= 2^32 "
                  "(device mirrors use u32 indices)");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    // kronecker.rs: b in a's storage (to_other_storage); a CSR mirror's CSC b uses its cache
    const sprs_b200_csmat* bb = b;
    sprs_b200_csmat* owned = nullptr;
    if (b->storage != a->storage) {
        if (a->storage == SPRS_B200_CSR) {
            SPRS_TRY(csmat_csr_view(ctx, b, &bb));
        } else {
            SPRS_TRY(sprs_b200_csmat_to_other_storage(ctx, b, &owned));
            bb = owned;
        }
    }
    const uint64_t outer_c = a->outer * bb->outer;
    sprs_b200_csmat* c = construct_result(ctx, a->storage, rows, cols, nnz);
    const KronOperands o{a->d_indptr, a->d_indices, a->d_data, bb->d_indptr, bb->d_indices,
                         bb->d_data, bb->outer, bb->inner, bb->nnz,
                         a->indptr_bytes == 8 ? 1u : 0u, bb->indptr_bytes == 8 ? 1u : 0u};
    int st = alloc_result(ctx, c, s);
    if (st == SPRS_B200_OK) {
        const uint64_t n_tiles = (nnz + CONSTRUCT_TILE - 1) / CONSTRUCT_TILE;
        const unsigned fill_grid = (unsigned)((n_tiles + 7) / 8);
        if (c->indptr_bytes == 4) {
            kron_indptr_kernel<uint32_t><<<grid_for(ctx, outer_c + 1), 256, 0, s>>>(
                o, outer_c, nnz, (uint32_t*)c->d_indptr);
            if (n_tiles)
                kron_fill_kernel<uint32_t><<<fill_grid, 256, 0, s>>>(
                    o, outer_c, nnz, n_tiles, (const uint32_t*)c->d_indptr, c->d_indices,
                    c->d_data);
        } else {
            kron_indptr_kernel<uint64_t><<<grid_for(ctx, outer_c + 1), 256, 0, s>>>(
                o, outer_c, nnz, (uint64_t*)c->d_indptr);
            if (n_tiles)
                kron_fill_kernel<uint64_t><<<fill_grid, 256, 0, s>>>(
                    o, outer_c, nnz, n_tiles, (const uint64_t*)c->d_indptr, c->d_indices,
                    c->d_data);
        }
        ctx->launches += n_tiles ? 2 : 1;
        if (cudaGetLastError() != cudaSuccess) {
            sprs_b200_set_error(ctx, "kron: launch failed");
            st = SPRS_B200_ERR_CUDA;
        } else {
            st = finish_result(ctx, c, s, "kron");
        }
    }
    if (owned) sprs_b200_csmat_free(owned);
    if (st != SPRS_B200_OK) {
        sprs_b200_csmat_free(c);
        return st;
    }
    *out = c;
    return SPRS_B200_OK;
}

int sprs_b200_csmat_transpose_view(sprs_b200_ctx* ctx, const sprs_b200_csmat* m,
                                   sprs_b200_csmat** out) {
    if (!ctx || !m || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    auto* t = new sprs_b200_csmat();
    t->ctx = ctx;
    t->storage = m->storage == SPRS_B200_CSR ? SPRS_B200_CSC : SPRS_B200_CSR;
    t->rows = m->cols;
    t->cols = m->rows;
    t->outer = m->outer;
    t->inner = m->inner;
    t->nnz = m->nnz;
    t->indptr_bytes = m->indptr_bytes;
    t->d_indptr = m->d_indptr;
    t->d_indices = m->d_indices;
    t->d_data = m->d_data;
    t->owns = false;
    int st = spmv_prepare(ctx, t, ctx->stream, false);
    if (st == SPRS_B200_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
        sprs_b200_set_error(ctx, "transpose_view: partition kernel failed");
        st = SPRS_B200_ERR_CUDA;
    }
    if (st != SPRS_B200_OK) {
        sprs_b200_csmat_free(t);
        return st;
    }
    *out = t;
    return SPRS_B200_OK;
}

}  // extern "C"
