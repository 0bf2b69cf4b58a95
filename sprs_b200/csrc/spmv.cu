// spmv.cu -- CSR x dense-vector product for sm_90a (H100).
//
// Replaces prod::mul_acc_mat_vec_csr (sprs/src/sparse/prod.rs:103-127) and the
// one-column case of prod::csr_mulacc_dense_colmaj (prod.rs:274-298), which is what
// `&A * &x` runs (sprs/src/sparse/csmat.rs:2142-2148).
//
// Design (DESIGN.md 4.1).  The kernel is bound by the x gathers -- the L1TEX pipe, the L1 lines
// in-flight gathers hold, and the 32-byte sector each 8-byte x element pulls through L2 -- not by
// HBM: "ceiling" kernels (the same streams and gathers with the row logic removed;
// tools/spmv_lab.cu, csrc/diag.cu) stay well below the HBM roofline whatever the staging.  So:
//   * MERGE-PATH TILES: the CSR stream is cut where  nnz + 16 * (row ends)  reaches multiples of
//     1024 (tile_cut_kernel): a tile is ~900 non-zeros of long rows or at most 64 row ends of
//     empty ones, never a thousand rows for one warp.  A tile belongs to ONE WARP; warps are
//     persistent and autonomous (no CTA-wide barrier, no shared memory: the whole unified array
//     is L1 for the gathers);
//   * ROWS STRAIGHT FROM GLOBAL MEMORY, lanes matched to the rows (rows_direct): per block of 31
//     rows, tiny rows (<= 8 non-zeros) one lane each in storage order -- the reference's bits
//     where no tile carries the row, from y[r] when accumulating --, the others packed G = 4..32
//     lanes per row with 4 index / value / gather loads in
//     flight per lane and one G-lane butterfly per row, very long rows by the whole warp.
//     Nothing is staged, nothing but a row sum crosses lanes;
//   * loads: ld.global.nc.L1::no_allocate + L2 evict_first for the matrix (read exactly once),
//     ld.global.nc + L2 evict_last for x; 40 warps per SM hide the latency;
//   * the row cut by a tile end leaves its partial in carry[t]; a second tiny kernel adds the
//     carries in tile order (deterministic, no atomics);
//   * the multi-target flavour (fused all-gather of the multi-GPU path, DESIGN.md 5) also
//     delivers every finished row to the peers: a plain store into ONE multicast address, or --
//     several peer mappings -- the tile's rows staged in 528 bytes of shared memory per warp and
//     sent as one TMA bulk store per peer;
//   * HOT SET (large skewed matrices, spmv_prepare_hot): x of the K most-referenced columns is
//     staged in shared memory by every CTA (one 32-warp CTA per SM) and the kernel reads a
//     tagged copy of the index stream, so those gathers move no L2 sector.
// The summation order depends only on indptr and the cut constants, and y is bit-identical to
// tests/spmv_model.py (its host restatement) for any values.  Rows longer than 8 non-zeros and
// carried rows (y0 + partial + carries) agree with the reference to rounding (parity gate:
// |d| <= 1e-6 * sum|terms|, SURVEY 8d).  Arithmetic is MulAcc::mul_acc's (mul_acc.rs:28-30):
// unfused multiply, then add.
//
// Algorithmic bytes per nnz: 12 (8 data + 4 index) + 8 per row (y) -- the BASELINE roofline
// 12*nnz + 8*n; indptr (4 B/row), the tile cuts (16 B per tile) and x gathers are overhead.

#include "common.cuh"
#include "ptx.cuh"
#include "scan.cuh"

#include <algorithm>
#include <cstdlib>
#include <type_traits>

namespace {

// ---- partition: merge-path cuts.  A tile is W units of COST along the path that consumes the
// non-zeros and the row ends of the CSR stream, a row end counting ROW_COST non-zeros: the cut of
// tile t is the point (tile_row[t], tile_k[t]) with  k + ROW_COST * r = t * W,  r = the rows
// whose end has been passed, indptr[r] <= k <= indptr[r+1].  Equal-nnz tiles are not enough on an
// R-MAT matrix: its sparse tail has stretches of thousands of (nearly) empty rows, a 1024-nnz
// tile there holds ~1700 rows -- 55 dependent boundary fetches for one warp while the others
// wait.
// With the row cost in the cut a tile has at most W / ROW_COST row ends.
constexpr int SPMV_STAGE_ROWS = 66;  // fused all-gather: staged rows per warp tile (64 row ends + parity pad)
constexpr uint32_t SPMV_ROW_COST = 16;  // default; 2nd field of SPRS_B200_SPMV_VARIANT for tuning runs

template <typename P>
__global__ void tile_cut_kernel(const P* __restrict__ indptr, uint32_t rows, uint64_t nnz,
                                uint64_t n_tiles, uint32_t w, uint32_t row_cost,
                                uint32_t* __restrict__ tile_row, P* __restrict__ tile_k) {
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t > n_tiles) return;
    if (t == n_tiles) {  // the end of the path
        tile_row[t] = rows;
        tile_k[t] = (P)nnz;
        return;
    }
    const uint64_t d = t * (uint64_t)w;
    uint32_t lo = 0, hi = rows;  // largest r in [0, rows] with indptr[r] + ROW_COST * r <= d
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if ((uint64_t)indptr[mid] + (uint64_t)row_cost * mid <= d)
            lo = mid;
        else
            hi = mid - 1;
    }
    uint64_t k = d - (uint64_t)row_cost * lo;
    // the cut may fall inside the "row end" step of row lo: all its non-zeros are then consumed
    const uint64_t row_end = lo < rows ? (uint64_t)indptr[(size_t)lo + 1] : nnz;
    if (k > row_end) k = row_end;
    tile_row[t] = lo;
    tile_k[t] = (P)k;
}

// What the row emitters need.
struct RowSink {
    double* y;                  // this GPU's y (target 0)
    const SpmvTargets* yt;      // MULTI only: the kernel parameter itself (constant bank)
    double* carry_slot;
    uint32_t r1;                // first row NOT owned by the tile (== its carry row when < rows)
    int accumulate;
    // MULTI only: the tile's rows for the peers are STAGED in shared memory (row r at
    // stage[r - stage_off]) and leave as one TMA bulk store per target when the tile is done;
    // nullptr = every row is stored to the peers directly
    double* stage;
    uint32_t stage_off;
};
// y[r] is written to every target buffer: target 0 is this GPU's own y; targets 1.. are the
// peer GPUs' y buffers (CUDA IPC / VMM mappings) or the NVSwitch multicast address of y (fused
// SpMV + all-gather over NVLink: the result of a row leaves for the peers the moment it is
// reduced, overlapped with the rest of the kernel, instead of a separate collective afterwards).
// from_y: the sum already started from y[r] (tiny rows under accumulate), so it is stored as is.
template <bool MULTI>
__device__ __forceinline__ void sink_row(const RowSink& k, uint64_t r, double sum, bool from_y = false) {
    if (r < k.r1) {
        const double v = k.accumulate && !from_y ? __dadd_rn(k.y[r], sum) : sum;
        k.y[r] = v;
        if (MULTI) {
#pragma unroll
            if (k.stage) {
                k.stage[(uint32_t)r - k.stage_off] = v;
            } else {
#pragma unroll
                for (int q = 1; q < SPMV_MAX_TARGETS; ++q)
                    if (q < k.yt->n) k.yt->p[q][r] = v;
            }
        }
    } else {
        *k.carry_slot = sum;  // row continues in a later tile: spmv_fixup_kernel adds it
    }
}

// x[c] for an entry of the index stream.  On a mirror with a hot set the SpMV reads the TAGGED
// copy of the stream: a hot column is stored as HOT_TAG | slot and its x value comes from the
// CTA's shared-memory copy of the hot set instead of a gathered L2 sector.  The value is the
// same double either way, so every product and sum keeps its bits.
constexpr uint32_t HOT_TAG = 0x80000000u;
template <bool HOT>
__device__ __forceinline__ double gather_x(const double* __restrict__ x, const double* hot,
                                           uint32_t c, uint64_t polx) {
    if (HOT && (c & HOT_TAG)) return hot[c & ~HOT_TAG];
    return ldg_f64_hint(x + c, polx);
}

// Rows [r0, r_last] of one warp tile [k0, k1), straight from global memory -- index, value
// (L1::no_allocate, L2 evict_first) and the x gather (L2 evict_last), U of each in flight per
// lane; nothing is staged and nothing but a row sum crosses lanes (~1 instruction per non-zero on
// long rows).  Row boundaries come 31 rows at a time (lane L: indptr[rbase + L]), and every block
// of 31 rows is taken in three sweeps, because R-MAT blocks mix rows of 0, 5, 50 and 5000
// non-zeros and any single lanes-per-row choice leaves most lanes idle:
//   1. TINY rows (at most 2U = 8 non-zeros, empty rows included): every lane takes its own row,
//      all of them in one pass, summed in storage order (from y[r] when accumulating a row that
//      no tile carries: the reference's bits);
//   2. the other rows, packed (no slot is spent on a tiny row): G lanes per row, 32/G rows per
//      pass, each group walking its row with stride G; one G-lane butterfly finishes a row;
//   3. rows longer than 4 steps of their group: the whole warp, one row at a time.
template <typename P, int G, int U, bool MULTI, bool HOT>
__device__ __forceinline__ void rows_direct(const RowSink& k, const P* __restrict__ indptr,
                                            const uint32_t* __restrict__ indices,
                                            const double* __restrict__ data,
                                            const double* __restrict__ x, const double* hot, P k0, P k1,
                                            uint32_t r0, uint32_t r_last, P b_first,
                                            uint64_t pol_stream, uint64_t polx, int lane) {
    constexpr int NG = 32 / G;
    constexpr unsigned FULL = 0xffffffffu;
    static_assert(G >= 4, "tiny rows have their own sweep: groups start at 4 lanes");
    const int gid = lane / G, gl = lane % G;
    // (offsets are as wide as the indptr: 32 bits unless nnz >= 2^32; row indices are 32-bit)
    P b = b_first;  // boundaries of the first block were prefetched by the caller
    for (uint32_t rbase = r0;; rbase += 31) {
        if (rbase != r0) {
            const uint32_t rr = rbase + lane;  // r_last + 1 <= rows < 2^32: no wrap for rr <= r_last + 1
            b = (rr >= rbase && rr <= r_last + 1) ? indptr[rr] : (P)0;
        }
        const int nrows = (r_last - rbase + 1) < 31 ? (int)(r_last - rbase + 1) : 31;
        // this lane's own row (lane < nrows), clamped to the tile
        P ms = b, me = __shfl_down_sync(FULL, b, 1);
        ms = ms > k0 ? ms : k0;
        me = me < k1 ? me : k1;
        if (lane >= nrows || me < ms) me = ms;
        const bool tiny = lane < nrows && (me - ms) <= (P)(2 * U);
        // ---- sweep 1: tiny rows, one lane each, storage order.  Accumulating, a row that no tile
        // carries starts from y[r] -- ((y0 + p0) + p1) + ..., the reference's order -- and an empty
        // one keeps y's bits (-0.0 included).  Row r0 is the previous tile's carry row, except in
        // tile 0, the only tile that starts at (row 0, non-zero 0).
        // (accumulate is uniform: each form gets its own copy of the sweep, so the plain one has
        // no y load and keeps its 48 registers)
        const uint32_t rl = rbase + lane;
        auto tiny_sweep = [&](auto acc_tag) {
            constexpr bool ACC = decltype(acc_tag)::value;
            const bool from_y = ACC && tiny && rl < k.r1 && (rl > r0 || (r0 == 0 && k0 == 0));
            double acc = from_y ? k.y[rl] : 0.0;  // (empty rows: y = 0, or y + 0 for a carried row)
            if (__any_sync(FULL, tiny && me > ms)) {
#pragma unroll
                for (int st = 0; st < 2; ++st) {
                    const P q = ms + (P)(st * U);
                    uint32_t c[U];
                    double v[U], xv[U];
#pragma unroll
                    for (int u = 0; u < U; ++u)
                        c[u] = (tiny && q + (P)u < me) ? ldg_stream_u32(indices + q + (P)u, pol_stream) : 0u;
#pragma unroll
                    for (int u = 0; u < U; ++u)
                        v[u] = (tiny && q + (P)u < me) ? ldg_stream_f64(data + q + (P)u, pol_stream) : 0.0;
#pragma unroll
                    for (int u = 0; u < U; ++u)
                        xv[u] = (tiny && q + (P)u < me) ? gather_x<HOT>(x, hot, c[u], polx) : 0.0;
#pragma unroll
                    for (int u = 0; u < U; ++u)
                        if (tiny && q + (P)u < me) acc = __dadd_rn(acc, __dmul_rn(v[u], xv[u]));
                    if (!__any_sync(FULL, tiny && q + (P)U < me)) break;
                }
            }
            if (tiny) sink_row<MULTI>(k, (uint64_t)rbase + lane, acc, from_y);
        };
        if (k.accumulate)
            tiny_sweep(std::true_type{});
        else
            tiny_sweep(std::false_type{});
        // ---- sweeps 2 and 3: the other rows, NG at a time
        unsigned todo = __ballot_sync(FULL, lane < nrows && !tiny);
        while (todo) {
            int j = -1;  // row (within the block) of this lane's group
#pragma unroll
            for (int g = 0; g < NG; ++g) {
                if (todo) {
                    const int jj = __ffs(todo) - 1;
                    todo &= todo - 1;
                    if (gid == g) j = jj;
                }
            }
            const bool valid = j >= 0;
            const int js = valid ? j : 0;
            P s = __shfl_sync(FULL, b, js);
            P e = __shfl_sync(FULL, b, js + 1);
            s = s > k0 ? s : k0;
            e = e < k1 ? e : k1;
            if (!valid || e < s) e = s;
            // a row much longer than its group would hold the warp behind G lanes
            const bool is_long = (G < 32) && (e - s) > (P)(4 * G * U);
            double acc = 0.0;
            for (P q = s + gl; q < (is_long ? s : e); q += (P)(G * U)) {
                uint32_t c[U];
                double v[U], xv[U];
#pragma unroll
                for (int u = 0; u < U; ++u)
                    c[u] = q + (P)(u * G) < e ? ldg_stream_u32(indices + q + (P)(u * G), pol_stream) : 0u;
#pragma unroll
                for (int u = 0; u < U; ++u)
                    v[u] = q + (P)(u * G) < e ? ldg_stream_f64(data + q + (P)(u * G), pol_stream) : 0.0;
#pragma unroll
                for (int u = 0; u < U; ++u)
                    xv[u] = q + (P)(u * G) < e ? gather_x<HOT>(x, hot, c[u], polx) : 0.0;
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (q + (P)(u * G) < e) acc = __dadd_rn(acc, __dmul_rn(v[u], xv[u]));
            }
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(FULL, acc, o));
            if (gl == 0 && valid && !is_long) sink_row<MULTI>(k, (uint64_t)rbase + j, acc);
            if (G < 32) {
                unsigned pending = __ballot_sync(FULL, gl == 0 && is_long);
                while (pending) {
                    const int src = __ffs(pending) - 1;
                    pending &= pending - 1;
                    const P qs = __shfl_sync(FULL, s, src), qe = __shfl_sync(FULL, e, src);
                    const int jj = __shfl_sync(FULL, j, src);
                    double a2 = 0.0;
                    for (P q = qs + lane; q < qe; q += (P)(32 * U)) {
                        uint32_t c[U];
                        double v[U], xv[U];
#pragma unroll
                        for (int u = 0; u < U; ++u)
                            c[u] = q + (P)(u * 32) < qe ? ldg_stream_u32(indices + q + (P)(u * 32), pol_stream) : 0u;
#pragma unroll
                        for (int u = 0; u < U; ++u)
                            v[u] = q + (P)(u * 32) < qe ? ldg_stream_f64(data + q + (P)(u * 32), pol_stream) : 0.0;
#pragma unroll
                        for (int u = 0; u < U; ++u)
                            xv[u] = q + (P)(u * 32) < qe ? gather_x<HOT>(x, hot, c[u], polx) : 0.0;
#pragma unroll
                        for (int u = 0; u < U; ++u)
                            if (q + (P)(u * 32) < qe) a2 = __dadd_rn(a2, __dmul_rn(v[u], xv[u]));
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) a2 = __dadd_rn(a2, __shfl_xor_sync(FULL, a2, o));
                    if (lane == 0) sink_row<MULTI>(k, (uint64_t)rbase + jj, a2);
                }
            }
        }
        if (r_last - rbase < 31) break;  // (also ends the loop when rbase + 31 would wrap)
    }
}

template <typename P, int NWARPS, int MINB, int U, bool MULTI, bool HOT>
__global__ void __launch_bounds__(NWARPS * 32, MINB)
    spmv_rows_kernel(const P* __restrict__ indptr, const uint32_t* __restrict__ indices,
                     const double* __restrict__ data, const uint32_t* __restrict__ tile_row,
                     const P* __restrict__ tile_k, const double* __restrict__ x,
                     const __grid_constant__ SpmvTargets yt,
                     double* __restrict__ carry, uint64_t nnz, uint32_t rows, uint32_t t_begin,
                     uint32_t t_end /* this launch covers tiles [t_begin, t_end) */, int accumulate,
                     uint64_t pol_stream /* L2 evict_first */, uint64_t polx /* L2 evict_last */,
                     int stage_rows /* MULTI: peers get their rows by TMA bulk stores (0: plain stores) */,
                     const uint32_t* __restrict__ hot_col /* HOT: the columns of the slots */,
                     uint32_t n_hot) {
    // (the two L2 policies are kernel PARAMETERS: warp-uniform by construction, so they live in
    // uniform registers; as per-thread createpolicy results every hinted load re-materialised
    // its descriptor)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // HOT: x of the hot columns, one copy per CTA in dynamic shared memory (`indices` is then
    // the tagged stream)
    extern __shared__ __align__(16) double hot_x[];
    if constexpr (HOT) {
        for (uint32_t q = threadIdx.x; q < n_hot; q += NWARPS * 32)
            hot_x[q] = ldg_f64_hint(x + hot_col[q], polx);
        __syncthreads();
    }
    const uint32_t GW = gridDim.x * NWARPS;
    RowSink sink;
    sink.y = yt.p[0];
    sink.yt = &yt;
    sink.accumulate = accumulate;
    sink.stage = nullptr;
    sink.stage_off = 0;
    // The peers' copies of y (fused all-gather).  A store per finished row and peer slows the
    // ISSUING kernel in proportion to rows x peers: remote stores queue in the LSU in front of
    // the loads.  With stage_rows set, the rows of a tile are staged in shared memory
    // (at most 64 row ends per tile = 512 bytes per warp) and leave through the TMA instead -- one
    // cp.async.bulk per target and tile.  Bulk copies need 16-byte alignment on both
    // sides: row r sits at stage[r + par - even base] with par = the parity of the peers' y
    // address (the launcher checked that all targets share it), an odd first / last row goes out
    // as a plain store.
    double* my_stage = nullptr;  // (the single-target kernel keeps all of the unified array as L1)
    if constexpr (MULTI) {
        __shared__ __align__(16) double stage_all[NWARPS * SPMV_STAGE_ROWS];
        my_stage = stage_all + warp * SPMV_STAGE_ROWS;
    }
    const uint32_t par = MULTI ? (uint32_t)(((uintptr_t)yt.p[1] >> 3) & 1) : 0u;
    uint32_t t = t_begin + blockIdx.x * NWARPS + warp;
    if (t >= t_end) return;
    // row range and the first 32 row boundaries of a tile are fetched ONE TILE AHEAD
    uint32_t r0 = tile_row[t], r1 = tile_row[t + 1];
    P k0 = tile_k[t], k1 = tile_k[t + 1];
    // lane L: indptr[r0 + L] while r0 + L <= r_last + 1 (r_last + 1 <= rows: always in range)
    P b_first = (uint64_t)r0 + lane <= (r1 < rows ? (uint64_t)r1 + 1 : (uint64_t)r1)
                    ? indptr[(size_t)r0 + lane] : (P)0;
    for (;;) {
        const uint32_t tn = t + GW;
        uint32_t r0n = 0, r1n = 0;
        P k0n = 0, k1n = 0;
        if (tn < t_end) {
            r0n = tile_row[tn];
            r1n = tile_row[tn + 1];
            k0n = tile_k[tn];
            k1n = tile_k[tn + 1];
        }
        sink.carry_slot = carry + t;
        sink.r1 = r1;
        if (MULTI && stage_rows) {
            // rows r0 .. r1-1 are the ones this tile delivers (r1 itself continues: carry)
            const uint32_t base = (r0 + par) & ~1u;  // even element index of the first staged slot
            const bool fits = r1 > r0 && (r1 + par - base) <= (uint32_t)SPMV_STAGE_ROWS;
            sink.stage = fits ? my_stage : nullptr;
            sink.stage_off = base - par;  // (wraps for r0 = 0, par = 1: r - stage_off is still r + 1)
            if (fits) {  // the previous tile's bulk stores must have READ the stage
                if (lane == 0) bulk_wait_group_read0();
                __syncwarp();
            }
        }
        const uint32_t r_last = r1 < rows ? r1 : r1 - 1;
        const uint64_t cnt = k1 - k0, nr = (uint64_t)(r_last - r0) + 1;  // mean row length = cnt / nr
#define SPMV_ROWS(G)                                                                            \
    rows_direct<P, G, U, MULTI, HOT>(sink, indptr, indices, data, x, hot_x, k0, k1, r0, r_last,   \
                                     b_first, pol_stream, polx, lane)
        if (cnt <= 24 * nr)
            SPMV_ROWS(4);
        else if (cnt <= 48 * nr)
            SPMV_ROWS(8);
        else if (cnt <= 96 * nr)
            SPMV_ROWS(16);
        else
            SPMV_ROWS(32);
#undef SPMV_ROWS
        if (MULTI && sink.stage) {
            fence_proxy_async();  // the lanes' stage writes -> visible to the async proxy
            __syncwarp();
            if (lane == 0) {
                uint32_t lo = r0, hi = r1;
                if ((lo + par) & 1u) {  // odd first row: plain store
                    const double v = my_stage[lo - sink.stage_off];
                    for (int q = 1; q < yt.n; ++q) yt.p[q][lo] = v;
                    ++lo;
                }
                if ((hi - lo) & 1u) {  // odd count: the last row as a plain store
                    --hi;
                    const double v = my_stage[hi - sink.stage_off];
                    for (int q = 1; q < yt.n; ++q) yt.p[q][hi] = v;
                }
                if (hi > lo) {
                    for (int q = 1; q < yt.n; ++q)
                        bulk_s2g(yt.p[q] + lo, my_stage + (lo - sink.stage_off), (hi - lo) * 8u);
                    bulk_commit_group();
                }
            }
            sink.stage = nullptr;
        }
        if (tn >= t_end) break;
        const P b_next = (uint64_t)r0n + lane <= (r1n < rows ? (uint64_t)r1n + 1 : (uint64_t)r1n)
                             ? indptr[(size_t)r0n + lane] : (P)0;
        t = tn;
        r0 = r0n;
        r1 = r1n;
        k0 = k0n;
        k1 = k1n;
        b_first = b_next;
    }
    if (MULTI && stage_rows && lane == 0) bulk_wait_group0();  // performed before the grid retires
}

// carries: tile t left the partial sum of row tile_row[t+1] in carry[t]; consecutive
// tiles with the same carry row form a run that is summed in tile order by its head.
__global__ void spmv_fixup_kernel(const uint32_t* __restrict__ tile_row,
                                  const double* __restrict__ carry, SpmvTargets yt,
                                  uint64_t n_tiles) {
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t + 1 >= n_tiles) return;
    const uint32_t row = tile_row[t + 1];
    if (t > 0 && tile_row[t] == row) return;  // not the head of its run
    // tile_row is sorted: the run [t, end) of tiles whose carry row is `row` ends at the
    // first u with tile_row[u + 1] > row.  Gallop + binary search, then a load-independent sum
    // in tile order (a hub row of 1e6 non-zeros is a run of thousands of tiles).
    uint64_t lo = t + 1, hi = n_tiles - 1;  // candidates for `end` (carry rows exist for u < n_tiles-1)
    for (uint64_t step = 1; lo + step < hi; step <<= 1) {
        if (tile_row[lo + step + 1] > row) {
            hi = lo + step;
            break;
        }
        lo += step;
    }
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (tile_row[mid + 1] > row)
            hi = mid;
        else
            lo = mid + 1;
    }
    double sum = carry[t];
#pragma unroll 8
    for (uint64_t u = t + 1; u < lo; ++u) sum = __dadd_rn(sum, carry[u]);
    const double v = __dadd_rn(yt.p[0][row], sum);
#pragma unroll
    for (int q = 0; q < SPMV_MAX_TARGETS; ++q)
        if (q < yt.n) yt.p[q][row] = v;
}

// Carries of the row that ends in tile u (u >= 1): the run of tiles [t, u-1] whose carry
// row is tile_row[u] left partial sums in carry[]; they are added in tile order, exactly
// like spmv_fixup_kernel does from the head of the run (same bits).
__device__ __forceinline__ void apply_carries_ending_in(const uint32_t* __restrict__ tile_row,
                                                        const double* carry, double* y,
                                                        uint64_t u) {
    const uint32_t row = tile_row[u];
    if (tile_row[u + 1] == row) return;  // the row continues past tile u: not final yet
    // head of the run: first index f in [1, u] with tile_row[f] >= row, t = f - 1
    uint64_t hi = u, lo = 1;
    for (uint64_t step = 1; step < hi; step <<= 1) {  // gallop down: most runs are 1 tile
        if (tile_row[hi - step] < row) {
            lo = hi - step + 1;
            break;
        }
        hi -= step;
    }
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (tile_row[mid] >= row)
            hi = mid;
        else
            lo = mid + 1;
    }
    double sum = __ldcg(carry + lo - 1);
    for (uint64_t v = lo; v < u; ++v) sum = __dadd_rn(sum, __ldcg(carry + v));
    y[row] = __dadd_rn(__ldcg(y + row), sum);
}

__global__ void spmv_fixup_range_kernel(const uint32_t* __restrict__ tile_row, const double* carry,
                                        double* y, uint64_t u_lo, uint64_t u_hi) {
    const uint64_t u = u_lo + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (u >= 1 && u < u_hi) apply_carries_ending_in(tile_row, carry, y, u);
}

// ---- launch configuration ---------------------------------------------------------
// One kernel configuration ships: 8-warp CTAs, 5 per SM (= __launch_bounds__ minBlocks: the
// register budget; the kernel hides latency with warps, not registers), 4 loads of each kind in
// flight per lane (48 registers on sm_90a, no spills).  The two numbers of the CUT stay tunable
// for experiments:
// SPRS_B200_SPMV_VARIANT="w,row_cost" (cost units per tile, cost of a row end in non-zeros;
// read once per process -- they are baked into every mirror's tile arrays).
struct SpmvVariant {
    int wt, row_cost;
};
SpmvVariant spmv_variant() {
    static SpmvVariant v = [] {
        SpmvVariant d{1024, (int)SPMV_ROW_COST};
        if (const char* e = getenv("SPRS_B200_SPMV_VARIANT")) {
            int a, rc = (int)SPMV_ROW_COST;
            const int got = sscanf(e, "%d,%d", &a, &rc);
            if (got >= 1 && a >= 64 && rc >= 0) d = SpmvVariant{a, rc};
        }
        return d;
    }();
    return v;
}

constexpr int SPMV_NWARPS = 8, SPMV_CTAS_PER_SM = 5, SPMV_LOADS_IN_FLIGHT = 4;

// ---- hot set: the most-referenced columns of x, served from shared memory --------------
// R-MAT columns are heavily skewed: a few thousand columns take a large share of the non-zeros,
// but every gather of one of them still moves a 32-byte L2 sector into an L1 that cold gathers
// keep evicting.  A mirror with a hot set carries the K most-referenced columns (hot_col) and a
// tagged copy of its index stream for the SpMV (hot_idx: HOT_TAG | slot for a hot column); every
// CTA stages x of the hot columns in shared memory at kernel start.  The hot-set kernel runs
// fewer, larger CTAs, because each CTA holds one copy: one 32-warp CTA per SM (64 registers, no
// spills).  Measured on config 5 (DESIGN.md 4.1): K = 24576 beat 12288 and 16384, and two 20-warp
// CTAs per SM with 8192 slots each were slower (and spill at their 48-register budget).
constexpr int SPMV_HOT_NWARPS = 32, SPMV_HOT_CTAS_PER_SM = 1;
constexpr uint32_t SPMV_HOT_SLOTS = 24576;       // K of `auto` (192 KB of x per CTA)
constexpr uint32_t SPMV_HOT_MAX_SLOTS = 26624;   // 208 KB + the MULTI stage fit one CTA
// `auto` builds the hot set only where it pays: enough non-zeros to hide the staging of K
// values per CTA and launch, and a hot set that serves a real share of them (a uniform matrix
// like BASELINE config 2 has ~1 %).
constexpr uint64_t SPMV_HOT_MIN_NNZ = 1ull << 25;
constexpr double SPMV_HOT_MIN_SHARE = 0.10;

// SPRS_B200_SPMV_HOT=auto|0|K (read once per process): `auto` (default) = K = SPMV_HOT_SLOTS
// where the thresholds above hold; 0 = never; K = a hot set of K slots on every CSR mirror that
// can have one (A/B runs and tests).
struct SpmvHot {
    uint32_t k;
    bool forced;
};
SpmvHot spmv_hot() {
    static SpmvHot h = [] {
        SpmvHot d{SPMV_HOT_SLOTS, false};
        const char* e = getenv("SPRS_B200_SPMV_HOT");
        if (e && strcmp(e, "auto") != 0) {
            const long k = atol(e);
            d = SpmvHot{(uint32_t)(k < 0 ? 0 : k > (long)SPMV_HOT_MAX_SLOTS ? SPMV_HOT_MAX_SLOTS : k), true};
        }
        return d;
    }();
    return h;
}

template <typename P, bool MULTI, bool HOT>
auto* spmv_kernel() {
    constexpr int U = SPMV_LOADS_IN_FLIGHT;
    if constexpr (HOT)
        return spmv_rows_kernel<P, SPMV_HOT_NWARPS, SPMV_HOT_CTAS_PER_SM, U, MULTI, true>;
    else
        return spmv_rows_kernel<P, SPMV_NWARPS, SPMV_CTAS_PER_SM, U, MULTI, false>;
}

template <typename P>
int launch_variant(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x,
                   const SpmvTargets& yt, int accumulate, uint64_t t0, uint64_t t1,
                   cudaStream_t s) {
    if (m->n_tiles >= 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_UNSUPPORTED, "spmv: more than 2^32 tiles");
    const bool multi = yt.n > 1, hot = m->n_hot > 0;
    auto kern = hot ? (multi ? spmv_kernel<P, true, true>() : spmv_kernel<P, false, true>())
                    : (multi ? spmv_kernel<P, true, false>() : spmv_kernel<P, false, false>());
    const int nwarps = hot ? SPMV_HOT_NWARPS : SPMV_NWARPS;
    const int ctas = hot ? SPMV_HOT_CTAS_PER_SM : SPMV_CTAS_PER_SM;
    static bool configured_flags[64][4] = {};  // function attributes are per device
    bool& configured = configured_flags[ctx->device & 63][(multi ? 1 : 0) + (hot ? 2 : 0)];
    if (!configured) {
        int carve;
        if (hot) {
            // room for the largest hot set this process builds, in every CTA of the SM
            // (+ the multi-target stage, + the 1 KB the hardware reserves per CTA)
            const int dyn = (int)(spmv_hot().k * sizeof(double));
            const int per_cta = dyn + (multi ? nwarps * SPMV_STAGE_ROWS * 8 : 0) + 1024;
            SPRS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
            carve = (int)((100ull * ctas * per_cta + 228 * 1024 - 1) / (228 * 1024));
        } else {
            // no shared memory at all: the whole unified array is L1 for the gathers (every
            // in-flight gather holds an L1 line)
            // (the multi-target kernel stages 4.1 KB per CTA for its TMA stores: 5 CTAs need 26 KB)
            carve = multi ? 15 : 0;
            if (const char* e = getenv("SPRS_B200_SPMV_CARVEOUT")) carve = atoi(e);
        }
        SPRS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                                            carve));
        configured = true;
    }
    // How the peers get their rows:
    //   * several peer mappings (CUDA IPC / VMM, world-1 targets): staged per tile and sent by
    //     TMA bulk stores instead of a store per row and target;
    //   * ONE multicast target: a plain store per row (one store per row is cheap enough, and
    //     the staged form waits on the TMA between tiles).
    // Staging also needs all targets to agree on the 16-byte parity of their address.
    // SPRS_B200_SPMV_PEER_STORES=direct|tma forces one form (read per launch:
    // tools/scale_modes.py times both).
    int stage_rows = 0;
    if (multi) {
        stage_rows = yt.n > 2 ? SPMV_STAGE_ROWS : 0;
        if (const char* e = getenv("SPRS_B200_SPMV_PEER_STORES")) {
            if (e[0] == 'd') stage_rows = 0;
            if (e[0] == 't') stage_rows = SPMV_STAGE_ROWS;
        }
        for (int q = 2; q < yt.n; ++q)
            if ((((uintptr_t)yt.p[q] ^ (uintptr_t)yt.p[1]) >> 3) & 1) stage_rows = 0;
    }
    uint64_t grid = (uint64_t)ctx->sm_count * ctas;
    const uint64_t need = (t1 - t0 + nwarps - 1) / nwarps;
    if (grid > need) grid = need;
    const size_t smem = hot ? m->n_hot * sizeof(double) : 0;
    kern<<<(unsigned)grid, nwarps * 32, smem, s>>>((const P*)m->d_indptr,
                                                   hot ? m->d_hot_idx : m->d_indices,
                                                   m->d_data, m->d_tile_row, (const P*)m->d_tile_k, d_x, yt,
                                                   m->d_carry,
                                                   m->nnz, (uint32_t)m->rows, (uint32_t)t0,
                                                   (uint32_t)t1, accumulate, ctx->pol_evict_first,
                                                   ctx->pol_evict_last, stage_rows, m->d_hot_col,
                                                   m->n_hot);
    return SPRS_B200_OK;
}

// ---- hot-set construction (spmv_prepare) --------------------------------------------
// Warp-aggregated increment: the lanes holding the same key add once (the top column of an
// R-MAT matrix is referenced ~1e6 times).  `active` = the lanes taking part.
__device__ __forceinline__ void add_aggregated(uint32_t* counts, uint32_t key, unsigned active) {
    const unsigned peers = __match_any_sync(active, key);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(counts + key, (uint32_t)__popc(peers));
}

// counts[c] = references of column c in the index stream
__global__ void hot_count_kernel(const uint32_t* __restrict__ indices, uint64_t nnz,
                                 uint32_t* __restrict__ counts) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x + (threadIdx.x & ~31u); base < nnz;
         base += stride) {
        const uint64_t i = base + (threadIdx.x & 31);
        const bool valid = i < nnz;
        const unsigned active = __ballot_sync(0xffffffffu, valid);
        if (valid) add_aggregated(counts, indices[i], active);
    }
}

// Radix select of the K-th largest count, 16 bits at a time.  hi == ~0u: every referenced
// column, binned by the upper 16 bits of its count; otherwise the columns whose count has `hi`
// in its upper bits, binned by the lower 16.
__global__ void hot_count_hist_kernel(const uint32_t* __restrict__ counts, uint32_t cols,
                                      uint32_t hi, uint32_t* __restrict__ hist) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x + (threadIdx.x & ~31u); base < cols;
         base += stride) {
        const uint64_t i = base + (threadIdx.x & 31);
        const uint32_t c = i < cols ? counts[i] : 0u;
        const bool take = c > 0 && (hi == ~0u || (c >> 16) == hi);
        const unsigned active = __ballot_sync(0xffffffffu, take);
        if (take) add_aggregated(hist, hi == ~0u ? c >> 16 : c & 0xffffu, active);
    }
}

// The K hot columns: every count above `thr`, then the first `ties` columns (in column order)
// whose count equals it.  tie_rank == nullptr: flag the ties themselves (their scan is the rank)
__global__ void hot_flag_kernel(const uint32_t* __restrict__ counts, uint32_t cols, uint32_t thr,
                                const uint32_t* __restrict__ tie_rank, uint32_t ties,
                                uint8_t* __restrict__ flag) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= cols) return;
    const uint32_t c = counts[i];
    flag[i] = tie_rank ? (c > thr || (c == thr && tie_rank[i] < ties)) : c == thr;
}

// counts -> the tag map (a column's entry in the SpMV's index stream), hot_col[slot] = column,
// hot_nnz = the references the hot set serves
__global__ void hot_map_kernel(uint32_t* __restrict__ counts_map, uint32_t cols,
                               const uint8_t* __restrict__ sel, const uint32_t* __restrict__ slot,
                               uint32_t* __restrict__ hot_col, unsigned long long* hot_nnz) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= cols) return;
    if (sel[i]) {
        const uint32_t q = slot[i];
        atomicAdd(hot_nnz, (unsigned long long)counts_map[i]);
        hot_col[q] = (uint32_t)i;
        counts_map[i] = HOT_TAG | q;
    } else {
        counts_map[i] = (uint32_t)i;
    }
}

__global__ void hot_tag_kernel(const uint32_t* __restrict__ indices, uint64_t nnz,
                               const uint32_t* __restrict__ map, uint32_t* __restrict__ tagged) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz; i += stride)
        tagged[i] = map[indices[i]];
}

// Builds m's hot set, or leaves the mirror without one (n_hot = 0) where `auto` says it does not
// pay or a buffer cannot be allocated -- the SpMV then runs exactly as without it.
int spmv_prepare_hot(sprs_b200_ctx* ctx, sprs_b200_csmat* m, cudaStream_t s) {
    const SpmvHot cfg = spmv_hot();
    if (cfg.k == 0 || m->nnz == 0 || m->cols == 0 || m->cols >= HOT_TAG) return SPRS_B200_OK;
    if (!cfg.forced && m->nnz < SPMV_HOT_MIN_NNZ) return SPRS_B200_OK;
    const uint32_t cols = (uint32_t)m->cols;
    const unsigned grid_nnz =
        (unsigned)std::min<uint64_t>((m->nnz + 255) / 256, (uint64_t)ctx->sm_count * 16);
    const unsigned grid_cols = (unsigned)((cols + 255) / 256);
    // (returns OK with m->n_hot still 0 wherever the mirror gets no hot set; a buffer that cannot
    // be allocated means no hot set, not an error)
    Owned<uint32_t> counts, hist, slot, hot_col, hot_idx;
    Owned<uint8_t> flag;
    Owned<unsigned long long> d_hot_nnz;
    if (counts.alloc(ctx, cols * sizeof(uint32_t), "spmv hot set") != SPRS_B200_OK ||
        hist.alloc(ctx, 65536 * sizeof(uint32_t), "spmv hot set") != SPRS_B200_OK ||
        flag.alloc(ctx, cols, "spmv hot set") != SPRS_B200_OK ||
        slot.alloc(ctx, (cols + 1ull) * sizeof(uint32_t), "spmv hot set") != SPRS_B200_OK ||
        d_hot_nnz.alloc(ctx, sizeof(unsigned long long), "spmv hot set") != SPRS_B200_OK)
        return SPRS_B200_OK;
    // ---- references per column, then the count of the K-th most referenced column
    SPRS_CUDA(ctx, cudaMemsetAsync(counts, 0, cols * sizeof(uint32_t), s));
    SPRS_CUDA(ctx, cudaMemsetAsync(hist, 0, 65536 * sizeof(uint32_t), s));
    SPRS_CUDA(ctx, cudaMemsetAsync(d_hot_nnz, 0, sizeof(unsigned long long), s));
    hot_count_kernel<<<grid_nnz, 256, 0, s>>>(m->d_indices, m->nnz, counts);
    hot_count_hist_kernel<<<grid_cols, 256, 0, s>>>(counts, cols, ~0u, hist);
    ctx->launches += 2;
    std::vector<uint32_t> h(65536);
    SPRS_CUDA(ctx, cudaMemcpyAsync(h.data(), hist, 65536 * sizeof(uint32_t),
                                   cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    uint64_t above = 0, referenced = 0;
    for (uint32_t b = 0; b < 65536; ++b) referenced += h[b];
    uint32_t k = cfg.k, thr = 1, ties = 0xffffffffu;  // K or fewer referenced columns: all
    if (referenced > k) {
        uint32_t bhi = 65535;  // (the loops stop: the bins hold more than K columns)
        while (above + h[bhi] < k) above += h[bhi--];
        SPRS_CUDA(ctx, cudaMemsetAsync(hist, 0, 65536 * sizeof(uint32_t), s));
        hot_count_hist_kernel<<<grid_cols, 256, 0, s>>>(counts, cols, bhi, hist);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaMemcpyAsync(h.data(), hist, 65536 * sizeof(uint32_t),
                                       cudaMemcpyDeviceToHost, s));
        SPRS_CUDA(ctx, cudaStreamSynchronize(s));
        uint32_t blo = 65535;
        while (above + h[blo] < k) above += h[blo--];
        thr = (bhi << 16) | blo;
        ties = k - (uint32_t)above;  // columns of count thr to take, in column order
    } else {
        k = (uint32_t)referenced;
    }
    // ---- select, slots in column order, tag map
    hot_flag_kernel<<<grid_cols, 256, 0, s>>>(counts, cols, thr, nullptr, 0, flag);
    ctx->launches += 1;
    SPRS_TRY((device_exclusive_scan<uint8_t, uint32_t>(ctx, flag, cols, slot, s)));
    hot_flag_kernel<<<grid_cols, 256, 0, s>>>(counts, cols, thr, slot, ties, flag);
    ctx->launches += 1;
    SPRS_TRY((device_exclusive_scan<uint8_t, uint32_t>(ctx, flag, cols, slot, s)));
    if (hot_col.alloc(ctx, k * sizeof(uint32_t), "spmv hot set") != SPRS_B200_OK)
        return SPRS_B200_OK;
    hot_map_kernel<<<grid_cols, 256, 0, s>>>(counts, cols, flag, slot, hot_col, d_hot_nnz);
    ctx->launches += 1;
    unsigned long long hot_nnz = 0;
    SPRS_CUDA(ctx, cudaMemcpyAsync(&hot_nnz, d_hot_nnz, sizeof(hot_nnz), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    if (!cfg.forced && (double)hot_nnz < SPMV_HOT_MIN_SHARE * (double)m->nnz) return SPRS_B200_OK;
    // ---- the tagged index stream (+4 bytes per non-zero)
    if (hot_idx.alloc(ctx, m->nnz * sizeof(uint32_t) + 16, "spmv hot set") != SPRS_B200_OK)
        return SPRS_B200_OK;
    hot_tag_kernel<<<grid_nnz, 256, 0, s>>>(m->d_indices, m->nnz, counts, hot_idx);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    SPRS_CUDA(ctx, cudaGetLastError());
    m->d_hot_col = hot_col.release();
    m->d_hot_idx = hot_idx.release();
    m->n_hot = k;
    return SPRS_B200_OK;
}

int check_spmv_args(sprs_b200_ctx* ctx, const sprs_b200_csmat* m) {
    if (m->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch: spmv needs a CSR mirror");
    if (!m->d_tile_row) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "csmat has no SpMV partition");
    return SPRS_B200_OK;
}

}  // namespace

int spmv_tile_nnz() { return spmv_variant().wt; }

int spmv_prepare(sprs_b200_ctx* ctx, sprs_b200_csmat* m, cudaStream_t s, bool hot_set) {
    if (m->storage != SPRS_B200_CSR) return SPRS_B200_OK;  // CSC mirrors are converted first
    const uint32_t w = (uint32_t)spmv_tile_nnz();  // cost units per tile
    const uint32_t row_cost = (uint32_t)spmv_variant().row_cost;
    const uint64_t total = m->nnz + (uint64_t)row_cost * m->rows;
    m->n_tiles = total == 0 ? 1 : (total + w - 1) / w;
    SPRS_TRY(mem_alloc(ctx, MemKind::device, (m->n_tiles + 1) * sizeof(uint32_t), nullptr,
                       "spmv partition", (void**)&m->d_tile_row));
    SPRS_TRY(mem_alloc(ctx, MemKind::device, (m->n_tiles + 1) * (size_t)m->indptr_bytes, nullptr,
                       "spmv partition", &m->d_tile_k));
    SPRS_TRY(mem_alloc(ctx, MemKind::device, m->n_tiles * sizeof(double), nullptr,
                       "spmv partition", (void**)&m->d_carry));
    const uint64_t n = m->n_tiles + 1;
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (m->indptr_bytes == 4)
        tile_cut_kernel<uint32_t><<<grid, 256, 0, s>>>((const uint32_t*)m->d_indptr, (uint32_t)m->rows,
                                                       m->nnz, m->n_tiles, w, row_cost, m->d_tile_row,
                                                       (uint32_t*)m->d_tile_k);
    else
        tile_cut_kernel<uint64_t><<<grid, 256, 0, s>>>((const uint64_t*)m->d_indptr, (uint32_t)m->rows,
                                                       m->nnz, m->n_tiles, w, row_cost, m->d_tile_row,
                                                       (uint64_t*)m->d_tile_k);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    if (hot_set) SPRS_TRY(spmv_prepare_hot(ctx, m, s));
    return SPRS_B200_OK;
}

int spmv_launch_targets(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x,
                        const SpmvTargets& yt, int accumulate, cudaStream_t s) {
    SPRS_TRY(check_spmv_args(ctx, m));
    if (m->rows == 0) return SPRS_B200_OK;
    if (m->indptr_bytes == 4)
        SPRS_TRY(launch_variant<uint32_t>(ctx, m, d_x, yt, accumulate, 0, m->n_tiles, s));
    else
        SPRS_TRY(launch_variant<uint64_t>(ctx, m, d_x, yt, accumulate, 0, m->n_tiles, s));
    ctx->launches += 1;
    if (m->n_tiles > 1) {
        const unsigned fgrid = (unsigned)((m->n_tiles - 1 + 255) / 256);
        spmv_fixup_kernel<<<fgrid, 256, 0, s>>>(m->d_tile_row, m->d_carry, yt, m->n_tiles);
        ctx->launches += 1;
    }
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

// SpMV over tiles [t0, t1) followed by the carries of the rows that END in those tiles: once
// this has run for every tile below t1 (chunks in increasing order on one stream), rows
// [0, tile_row[t1]) of y are final -- the same sums in the same order as the one-shot
// spmv_launch (apply_carries_ending_in adds a run's carries in tile order from its head, like
// spmv_fixup_kernel).  Used to pipeline something behind finished row ranges (the D2H copy of
// the host path, api.cu).
int spmv_launch_tile_range(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x,
                           double* d_y, int accumulate, uint64_t t0, uint64_t t1,
                           cudaStream_t s) {
    SPRS_TRY(check_spmv_args(ctx, m));
    if (t1 > m->n_tiles || t0 >= t1) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "bad tile range");
    SpmvTargets yt;
    yt.n = 1;
    yt.p[0] = d_y;
    for (int q = 1; q < SPMV_MAX_TARGETS; ++q) yt.p[q] = nullptr;
    if (m->indptr_bytes == 4)
        SPRS_TRY(launch_variant<uint32_t>(ctx, m, d_x, yt, accumulate, t0, t1, s));
    else
        SPRS_TRY(launch_variant<uint64_t>(ctx, m, d_x, yt, accumulate, t0, t1, s));
    spmv_fixup_range_kernel<<<(unsigned)((t1 - t0 + 255) / 256), 256, 0, s>>>(
        m->d_tile_row, m->d_carry, d_y, t0, t1);
    ctx->launches += 2;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

int spmv_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x, double* d_y,
                int accumulate, cudaStream_t s) {
    SpmvTargets yt;
    yt.n = 1;
    yt.p[0] = d_y;
    for (int q = 1; q < SPMV_MAX_TARGETS; ++q) yt.p[q] = nullptr;
    return spmv_launch_targets(ctx, m, d_x, yt, accumulate, s);
}
