// binop.cu -- sparse + sparse, sparse - sparse, Hadamard product and scalar scale for sm_90a.
//
// Replaces csmat_binop / csmat_binop_same_storage_raw (sprs/src/sparse/binop.rs:178-271), which
// `&A + &B`, `&A - &B` and binop::mul_mat_same_storage run, and CsMatBase::map (csmat.rs:
// 1289-1305), which `&A * s` runs.  Every output entry is ONE IEEE operation on the operands --
// f(a, 0.0), f(0.0, b) or f(a, b) -- kept only when the result is not 0.0 (NaN is kept), so the
// result is bit-identical to the reference.
//
// Design (DESIGN.md 4.7).  The operation only knows outer and inner dimensions, so one code path
// serves CSR + CSR and CSC + CSC.  Work is cut along the merged (outer, inner) stream of both
// operands, like the SpMV's merge-path tiles:
//   * COST  w(i) = ipA[i] + ipB[i] + ROW_COST * i: an operand entry costs 1, an outer dimension's
//     end ROW_COST.  A tile is TILE cost units, a lane of the tile's warp LANE_COST of them, so a
//     lane handles at most 32 entries or 2 row ends: hub rows of 10^6 entries are spread over
//     thousands of lanes, runs of empty rows over as many lanes as they cost.
//   * CUT   at cost d: a binary search over rows (the largest r with w(r) <= d), then a
//     merge-path diagonal search on the two sorted index lists of row r (ties: A first).  The
//     split is SNAPPED so that an equal pair A[ja-1] == B[jb] is never separated: a `Both` is
//     always produced by one lane.  cut_kernel cuts the tile boundaries; every lane cuts its own
//     start and end inside its tile's bounds.
//   * COUNT pass: each lane walks its range, evaluates f and the zero test, and stores its kept
//     count.  SCAN (scan.cuh, 64-bit) of the lane counts gives every lane's output offset
//     directly: lanes walk the merged stream in order.  FILL pass: the same walk writes indices,
//     data and indptr[r+1] of every row that ends in the lane's range, empty rows included.
//     No atomics, no inter-CTA waits: the output is deterministic.
//   * Operand values are read with the L2 evict_first policy, indices through the read-only
//     path (both L1-allocating: a lane walks consecutive entries of each list); indptr may be
//     u32 or u64 independently for A, B and C.

#include "common.cuh"
#include "ptx.cuh"
#include "scan.cuh"

#include <algorithm>
#include <cstdlib>

namespace {

constexpr uint64_t BINOP_TILE = 1024;      // cost units per warp tile
constexpr uint64_t BINOP_LANE_COST = 32;   // cost units per lane (BINOP_TILE / 32)
constexpr uint64_t BINOP_ROW_COST = 16;    // cost of one outer dimension's end
constexpr uint32_t NO_INDEX = 0xffffffffu; // inner indices are < 2^32 - 1

struct Cut {
    uint64_t r, ka, kb;  // rows passed; entries of A and B consumed (global positions)
};

template <typename PA, typename PB>
struct Operands {
    const PA* ipA;
    const uint32_t* iA;
    const double* vA;
    const PB* ipB;
    const uint32_t* iB;
    const double* vB;
    uint64_t outer;
    uint64_t pol;  // L2 evict_first
};

template <typename PA, typename PB>
__device__ __forceinline__ uint64_t path_cost(const Operands<PA, PB>& o, uint64_t r) {
    return (uint64_t)o.ipA[r] + (uint64_t)o.ipB[r] + BINOP_ROW_COST * r;
}

// The cut at cost d.  Rows are searched in [rlo, rhi] (w(rlo) <= d); within row r the number of
// A entries consumed lies in [ja_lo, ja_hi] (bounds from the enclosing tile's cuts: the merge
// path is monotone).
template <typename PA, typename PB>
__device__ Cut cut_at(const Operands<PA, PB>& o, uint64_t d, uint64_t rlo, uint64_t rhi,
                      const Cut* lo_cut, const Cut* hi_cut) {
    while (rlo < rhi) {
        const uint64_t mid = rlo + (rhi - rlo + 1) / 2;
        if (path_cost(o, mid) <= d)
            rlo = mid;
        else
            rhi = mid - 1;
    }
    const uint64_t r = rlo;
    const uint64_t a0 = o.ipA[r], b0 = o.ipB[r];
    if (r == o.outer) return Cut{r, a0, b0};  // the end of the path
    const uint64_t la = (uint64_t)o.ipA[r + 1] - a0, lb = (uint64_t)o.ipB[r + 1] - b0;
    uint64_t k = d - (a0 + b0 + BINOP_ROW_COST * r);
    if (k > la + lb) k = la + lb;  // the cut falls inside the row's end: the row is consumed
    // merge path: ja = A entries among the first k of the merged row (A first on equal indices)
    uint64_t lo = k > lb ? k - lb : 0, hi = k < la ? k : la;
    if (lo_cut && lo_cut->r == r && lo_cut->ka - a0 > lo) lo = lo_cut->ka - a0;
    if (hi_cut && hi_cut->r == r && hi_cut->ka - a0 < hi) hi = hi_cut->ka - a0;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (o.iA[a0 + mid] <= o.iB[b0 + k - mid - 1])
            lo = mid + 1;
        else
            hi = mid;
    }
    const uint64_t ja = lo;
    uint64_t jb = k - ja;
    // snap: A[ja-1] consumed and its equal B[jb] not -> consume B[jb] too (one lane owns a Both)
    if (ja > 0 && jb < lb && o.iA[a0 + ja - 1] == o.iB[b0 + jb]) ++jb;
    return Cut{r, a0 + ja, b0 + jb};
}

__device__ __forceinline__ double apply_op(int op, double a, double b) {
    return op == SPRS_B200_BINOP_ADD ? __dadd_rn(a, b)
         : op == SPRS_B200_BINOP_SUB ? __dsub_rn(a, b)
                                     : __dmul_rn(a, b);
}

// Walk the merged stream from c0 to c1: f on every entry, the zero test, and (FILL) the stores
// of the kept entries and of indptr[r+1] for every row that ends before c1.  Returns the number
// of entries kept.
template <bool FILL, typename PA, typename PB, typename PC>
__device__ uint64_t walk(const Operands<PA, PB>& o, int op, Cut c0, Cut c1, uint64_t pos,
                         PC* __restrict__ ipC, uint32_t* __restrict__ iC, double* __restrict__ vC) {
    const uint64_t start = pos;
    uint64_t ka = c0.ka, kb = c0.kb;
    for (uint64_t r = c0.r;; ++r) {
        const bool last = r == c1.r;
        const uint64_t ea = last ? c1.ka : (uint64_t)o.ipA[r + 1];
        const uint64_t eb = last ? c1.kb : (uint64_t)o.ipB[r + 1];
        uint32_t ia = ka < ea ? __ldg(o.iA + ka) : NO_INDEX;
        uint32_t ib = kb < eb ? __ldg(o.iB + kb) : NO_INDEX;
        while (ka < ea || kb < eb) {
            uint32_t col;
            double v;
            if (ia < ib) {         // Left(a): f(a, 0.0)
                col = ia;
                v = apply_op(op, ldg_f64_hint(o.vA + ka, o.pol), 0.0);
                ++ka;
                ia = ka < ea ? __ldg(o.iA + ka) : NO_INDEX;
            } else if (ib < ia) {  // Right(b): f(0.0, b)
                col = ib;
                v = apply_op(op, 0.0, ldg_f64_hint(o.vB + kb, o.pol));
                ++kb;
                ib = kb < eb ? __ldg(o.iB + kb) : NO_INDEX;
            } else {               // Both(a, b): f(a, b)
                col = ia;
                v = apply_op(op, ldg_f64_hint(o.vA + ka, o.pol), ldg_f64_hint(o.vB + kb, o.pol));
                ++ka;
                ++kb;
                ia = ka < ea ? __ldg(o.iA + ka) : NO_INDEX;
                ib = kb < eb ? __ldg(o.iB + kb) : NO_INDEX;
            }
            if (v != 0.0) {  // `!is_zero()`: +-0.0 dropped, NaN kept
                if (FILL) {
                    iC[pos] = col;
                    vC[pos] = v;
                }
                ++pos;
            }
        }
        if (last) break;
        if (FILL) ipC[r + 1] = (PC)pos;
    }
    return pos - start;
}

template <typename PA, typename PB>
__global__ void binop_cut_kernel(Operands<PA, PB> o, uint64_t total, uint64_t n_tiles,
                                 uint32_t* __restrict__ cut_r, uint64_t* __restrict__ cut_a,
                                 uint64_t* __restrict__ cut_b) {
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t > n_tiles) return;
    const uint64_t d = t * BINOP_TILE < total ? t * BINOP_TILE : total;
    const Cut c = cut_at(o, d, 0, o.outer, (const Cut*)nullptr, (const Cut*)nullptr);
    cut_r[t] = (uint32_t)c.r;
    cut_a[t] = c.ka;
    cut_b[t] = c.kb;
}

// The cuts of this lane's range [d0, d1) inside tile t; false for a lane past the end.
template <typename PA, typename PB>
__device__ __forceinline__ bool lane_range(const Operands<PA, PB>& o, uint64_t total, uint64_t t,
                                           const uint32_t* cut_r, const uint64_t* cut_a,
                                           const uint64_t* cut_b, Cut* c0, Cut* c1) {
    const uint64_t lane = threadIdx.x & 31;
    const uint64_t d0 = t * BINOP_TILE + lane * BINOP_LANE_COST;
    if (d0 >= total) return false;
    const uint64_t d1 = d0 + BINOP_LANE_COST < total ? d0 + BINOP_LANE_COST : total;
    const Cut lo{cut_r[t], cut_a[t], cut_b[t]}, hi{cut_r[t + 1], cut_a[t + 1], cut_b[t + 1]};
    *c0 = lane == 0 ? lo : cut_at(o, d0, lo.r, hi.r, &lo, &hi);
    *c1 = d1 == (t + 1) * BINOP_TILE || d1 == total ? hi : cut_at(o, d1, lo.r, hi.r, &lo, &hi);
    return true;
}

template <typename PA, typename PB>
__global__ void __launch_bounds__(256)
    binop_count_kernel(Operands<PA, PB> o, int op, uint64_t total, uint64_t n_tiles,
                       const uint32_t* __restrict__ cut_r, const uint64_t* __restrict__ cut_a,
                       const uint64_t* __restrict__ cut_b, uint32_t* __restrict__ lane_cnt) {
    const uint64_t t = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (t >= n_tiles) return;
    Cut c0, c1;
    uint32_t n = 0;
    if (lane_range(o, total, t, cut_r, cut_a, cut_b, &c0, &c1))
        n = (uint32_t)walk<false, PA, PB, uint32_t>(o, op, c0, c1, 0, nullptr, nullptr, nullptr);
    lane_cnt[t * 32 + (threadIdx.x & 31)] = n;
}

template <typename PA, typename PB, typename PC>
__global__ void __launch_bounds__(256)
    binop_fill_kernel(Operands<PA, PB> o, int op, uint64_t total, uint64_t n_tiles,
                      const uint32_t* __restrict__ cut_r, const uint64_t* __restrict__ cut_a,
                      const uint64_t* __restrict__ cut_b, const uint64_t* __restrict__ lane_off,
                      PC* __restrict__ ipC, uint32_t* __restrict__ iC, double* __restrict__ vC) {
    const uint64_t t = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    if (t >= n_tiles) return;
    if (t == 0 && (threadIdx.x & 31) == 0) ipC[0] = 0;
    Cut c0, c1;
    if (lane_range(o, total, t, cut_r, cut_a, cut_b, &c0, &c1))
        walk<true, PA, PB, PC>(o, op, c0, c1, lane_off[t * 32 + (threadIdx.x & 31)], ipC, iC, vC);
}

// CsMatBase::map(|x| x * s): structure copied, data[k] * s, nothing dropped
template <typename P>
__global__ void scale_kernel(const P* __restrict__ ip, const uint32_t* __restrict__ idx,
                             const double* __restrict__ val, uint64_t outer, uint64_t nnz,
                             double s, uint64_t pol, P* __restrict__ ip_out,
                             uint32_t* __restrict__ idx_out, double* __restrict__ val_out) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz; i += stride) {
        idx_out[i] = ldg_stream_u32(idx + i, pol);
        val_out[i] = __dmul_rn(ldg_stream_f64(val + i, pol), s);
    }
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= outer; i += stride)
        ip_out[i] = ip[i];
}

template <typename PA, typename PB, typename PC>
void launch_fill(const Operands<PA, PB>& o, int op, uint64_t total, uint64_t n_tiles,
                 const uint32_t* cut_r, const uint64_t* cut_a, const uint64_t* cut_b,
                 const uint64_t* lane_off, sprs_b200_csmat* c, cudaStream_t s) {
    const unsigned grid = (unsigned)((n_tiles + 7) / 8);
    binop_fill_kernel<PA, PB, PC><<<grid, 256, 0, s>>>(o, op, total, n_tiles, cut_r, cut_a, cut_b,
                                                       lane_off, (PC*)c->d_indptr, c->d_indices,
                                                       c->d_data);
}

// Both passes for one (lhs, rhs) indptr width pair.
template <typename PA, typename PB>
int run_binop(sprs_b200_ctx* ctx, const sprs_b200_csmat* a, const sprs_b200_csmat* b, int op,
              cudaStream_t s, sprs_b200_csmat** out) {
    const Operands<PA, PB> o{(const PA*)a->d_indptr, a->d_indices, a->d_data,
                             (const PB*)b->d_indptr, b->d_indices, b->d_data,
                             a->outer, ctx->pol_evict_first};
    const uint64_t total = a->nnz + b->nnz + BINOP_ROW_COST * a->outer;
    const uint64_t n_tiles = (total + BINOP_TILE - 1) / BINOP_TILE;
    const uint64_t n_lanes = n_tiles * 32;
    uint64_t nnz_c = 0;
    Owned<uint32_t> cut_r, lane_cnt;
    Owned<uint64_t> cut_a, cut_b, lane_off;
    if (n_tiles) {
        SPRS_TRY(cut_r.alloc_async(ctx, (n_tiles + 1) * 4, s, "binop"));
        SPRS_TRY(cut_a.alloc_async(ctx, (n_tiles + 1) * 8, s, "binop"));
        SPRS_TRY(cut_b.alloc_async(ctx, (n_tiles + 1) * 8, s, "binop"));
        SPRS_TRY(lane_cnt.alloc_async(ctx, n_lanes * 4, s, "binop"));
        SPRS_TRY(lane_off.alloc_async(ctx, (n_lanes + 1) * 8, s, "binop"));
        binop_cut_kernel<PA, PB><<<(unsigned)((n_tiles + 1 + 255) / 256), 256, 0, s>>>(
            o, total, n_tiles, cut_r, cut_a, cut_b);
        binop_count_kernel<PA, PB><<<(unsigned)((n_tiles + 7) / 8), 256, 0, s>>>(
            o, op, total, n_tiles, cut_r, cut_a, cut_b, lane_cnt);
        ctx->launches += 2;
        SPRS_TRY((device_exclusive_scan<uint32_t, uint64_t>(ctx, lane_cnt, n_lanes, lane_off, s)));
        if (cudaMemcpyAsync(&nnz_c, lane_off + n_lanes, 8, cudaMemcpyDeviceToHost, s) !=
                cudaSuccess ||
            cudaStreamSynchronize(s) != cudaSuccess)
            SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "binop: count pass failed");
    }
    CsmatPtr c = new_result(ctx, a->storage, a->rows, a->cols, nnz_c, indptr_bytes_for(nnz_c),
                            Arrays::pooled);
    SPRS_TRY(alloc_result(ctx, c.get(), s, "binop"));
    if (n_tiles == 0) {  // no outer dimension: indptr = [0]
        if (cudaMemsetAsync(c->d_indptr, 0, c->indptr_bytes, s) != cudaSuccess)
            SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "binop: memset failed");
    } else if (c->indptr_bytes == 4) {
        launch_fill<PA, PB, uint32_t>(o, op, total, n_tiles, cut_r, cut_a, cut_b, lane_off, c.get(), s);
    } else {
        launch_fill<PA, PB, uint64_t>(o, op, total, n_tiles, cut_r, cut_a, cut_b, lane_off, c.get(), s);
    }
    ctx->launches += n_tiles ? 1 : 0;
    if (cudaGetLastError() != cudaSuccess) SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "binop: launch failed");
    return finish_result(ctx, c, s, "binop", false, out);
}

}  // namespace

extern "C" {

int sprs_b200_csmat_binop(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                          const sprs_b200_csmat* rhs, int op, sprs_b200_csmat** out) {
    if (!ctx || !lhs || !rhs || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if (op != SPRS_B200_BINOP_ADD && op != SPRS_B200_BINOP_SUB && op != SPRS_B200_BINOP_MUL)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "binop: unknown op %d", op);
    // binop.rs:195-199: shapes first, then storage
    if (lhs->rows != rhs->rows || lhs->cols != rhs->cols)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (lhs->storage != rhs->storage) SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool a64 = lhs->indptr_bytes == 8, b64 = rhs->indptr_bytes == 8;
    if (!a64 && !b64) return run_binop<uint32_t, uint32_t>(ctx, lhs, rhs, op, s, out);
    if (!a64 && b64) return run_binop<uint32_t, uint64_t>(ctx, lhs, rhs, op, s, out);
    if (a64 && !b64) return run_binop<uint64_t, uint32_t>(ctx, lhs, rhs, op, s, out);
    return run_binop<uint64_t, uint64_t>(ctx, lhs, rhs, op, s, out);
}

int sprs_b200_csmat_scale(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, double s_val,
                          sprs_b200_csmat** out) {
    if (!ctx || !m || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    CsmatPtr c = new_result(ctx, m->storage, m->rows, m->cols, m->nnz, m->indptr_bytes,
                            Arrays::pooled);
    SPRS_TRY(alloc_result(ctx, c.get(), s, "scale"));
    const uint64_t n = m->nnz > m->outer + 1 ? m->nnz : m->outer + 1;
    const unsigned grid = (unsigned)std::min<uint64_t>((n + 255) / 256,
                                                       (uint64_t)ctx->sm_count * 16);
    if (m->indptr_bytes == 4)
        scale_kernel<uint32_t><<<grid, 256, 0, s>>>(
            (const uint32_t*)m->d_indptr, m->d_indices, m->d_data, m->outer, m->nnz, s_val,
            ctx->pol_evict_first, (uint32_t*)c->d_indptr, c->d_indices, c->d_data);
    else
        scale_kernel<uint64_t><<<grid, 256, 0, s>>>(
            (const uint64_t*)m->d_indptr, m->d_indices, m->d_data, m->outer, m->nnz, s_val,
            ctx->pol_evict_first, (uint64_t*)c->d_indptr, c->d_indices, c->d_data);
    ctx->launches += 1;
    return finish_result(ctx, c, s, "scale", false, out);
}

}  // extern "C"
