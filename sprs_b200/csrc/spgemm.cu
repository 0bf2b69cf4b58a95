// spgemm.cu -- CSR x CSR sparse product for sm_90a (H100).
//
// Replaces smmp::mul_csr_csr / mul_csr_csr_with_workspace (sprs/src/sparse/smmp.rs:
// 196-416): the two-phase Bank-Douglas SMMP product behind `&A * &B`
// (sprs/src/sparse/csmat.rs:1866-1949).
//   symbolic (smmp.rs:81-131): pattern of every C row = union of the B rows selected
//            by the A row; the reference marks a dense `seen[B.cols]` array and sorts.
//   numeric  (smmp.rs:151-189): values through a dense accumulator `tmp[B.cols]`,
//            gathered in C's sorted column order.
// Contract kept bit-exactly: C is CSR, zero-based indptr, per-row ascending duplicate-
// free indices, structural zeros KEPT (no value test, smmp.rs:109-129; SURVEY F12).
//
// Device design (DESIGN.md "SpGEMM"): rows are independent, so each phase bins rows by
// work and gives every bin the cheapest accumulator that fits:
//   symbolic, by n_prod_i = sum_{k in A_i} nnz(B_k) (upper bound of nnz(C_i)):
//     <= 128   one warp per row, 256-slot hash set per warp in shared memory;
//     <= 8192  one CTA per row, up-to-16384-slot hash set in shared memory (64 KB);
//     larger   one CTA per row, dense bitmap over B.cols (shared memory when it fits
//              in 200 KB, else a global-memory slot) -- the "spill" path; this is the
//              reference's `seen` array, one bit per column.
//   exclusive scan of the row counts -> C.indptr; then
//   numeric, by nnz(C_i) (now known):
//     <= 128   one warp per row, 256-slot hash map; A's non-zeros are applied ONE AT A
//              TIME in storage order with the lanes across the B row, so every C value
//              is the reference's sequential unfused sum -> bit-identical values;
//     <= 1024  one CTA per row, hash map in shared memory (up to 2048 of its 8192 slots),
//              then an in-place bitonic sort by column;
//     larger   one CTA per row: <= 4096 A non-zeros, dense f64 accumulation in shared
//              memory one 16384-column panel at a time; more ("hub" rows), a dense f64
//              accumulator over B.cols in a global-memory slot (the reference's `tmp`) +
//              bitmap; extraction walks the bitmap in order, so the row comes out sorted,
//              and re-zeroes what it touched.
//   The CTA-per-row bins add in the reference's order too, without f64 atomics: rounds of
//   one A non-zero per warp, products staged in storage order and folded by one warp, long
//   B rows finished by the whole CTA in turn (ordered_round) -> every value, index and
//   indptr entry bit-identical to the reference, under any thread schedule.
// Algorithmic bytes (SURVEY 8d): 12*(nnzA + n_prod + nnzC) + 8*(rows+1).

#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "scan.cuh"

struct sprs_b200_spgemm {
    sprs_b200_ctx* ctx = nullptr;
    const sprs_b200_csmat* a = nullptr;  // borrowed: must outlive the plan
    const sprs_b200_csmat* b = nullptr;
    uint64_t rows = 0, cols = 0, nnz_c = 0, n_prod = 0;
    uint64_t* d_nprod = nullptr;  // [rows]
    uint32_t* d_cnt = nullptr;    // [rows] nnz(C_i)
    uint64_t* d_cptr = nullptr;   // [rows+1]
    uint32_t* d_lists = nullptr;  // [3*rows] row lists per bin
    uint32_t* d_counters = nullptr;  // [8]
};

namespace {

constexpr uint32_t EMPTY = 0xffffffffu;
constexpr int NT = 256;
constexpr int WARPS = NT / 32;
constexpr uint32_t SYM_S_MAX = 128, SYM_M_MAX = 8192;
constexpr uint32_t NUM_S_MAX = 128, NUM_M_MAX = 4096;
constexpr int S_SLOTS = 256;
constexpr uint32_t SYM_M_SLOTS = 16384, NUM_M_SLOTS = 8192;
constexpr uint64_t BITMAP_SMEM_MAX_COLS = 200ull * 1024 * 8;  // 200 KB of bits

// Routing and kernel shapes: the hash bins
// serve only the rows they are cheap for -- with a shared-memory bitmap the symbolic phase sends
// rows with n_prod > B.cols/256 to the bitmap kernel, the numeric phase rows with
// nnz(C_i) > 16 * n_panels to the panel kernel; groups of G warps share one B row when the A row
// is short (half of config 4's large rows have <= 8 A non-zeros) in the symbolic kernels; the
// symbolic bitmap kernel runs 1024 threads and keeps several 32-entry chunks of B in flight per
// warp: it is bound by the L2 round trip of the B stream, not by the shared-memory atomics.

// Warps that share one B row in the CTA-per-row kernels: the largest power of two G with
// G * na <= nwarps (1 when grouping is off or the A row has at least nwarps/2 non-zeros).
__device__ __forceinline__ int warps_per_brow(uint32_t na, int nwarps, int grouping) {
    int g = 1;
    if (grouping)
        while (2 * g <= nwarps && (uint32_t)(2 * g) * na <= (uint32_t)nwarps) g *= 2;
    return g;
}

__device__ __forceinline__ uint32_t hash_col(uint32_t c, uint32_t mask) {
    return (c * 2654435761u) & mask;
}

// find-or-insert `col` in an open-addressing table; returns slot, sets *fresh
__device__ __forceinline__ uint32_t table_insert(uint32_t* keys, uint32_t mask, uint32_t col,
                                                 bool* fresh) {
    uint32_t h = hash_col(col, mask);
    for (;;) {
        const uint32_t old = atomicCAS(&keys[h], EMPTY, col);
        if (old == EMPTY) {
            *fresh = true;
            return h;
        }
        if (old == col) {
            *fresh = false;
            return h;
        }
        h = (h + 1) & mask;
    }
}

// ---- n_prod per row (warp per row) ---------------------------------------------
__global__ void __launch_bounds__(NT)
    nprod_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                 const uint32_t* __restrict__ b_ip, uint32_t rows,
                 uint64_t* __restrict__ nprod) {
    const int lane = threadIdx.x & 31;
    const uint64_t w0 = (blockIdx.x * (uint64_t)NT + threadIdx.x) >> 5;
    const uint64_t nw = ((uint64_t)gridDim.x * NT) >> 5;
    for (uint64_t r = w0; r < rows; r += nw) {
        uint64_t s = 0;
        for (uint32_t k = a_ip[r] + lane, e = a_ip[r + 1]; k < e; k += 32) {
            const uint32_t br = a_idx[k];
            s += b_ip[br + 1] - b_ip[br];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) nprod[r] = s;
    }
}

// bin rows: lists[bin*rows + i]; bin 0 small, 1 medium, 2 large; zero-work rows get cnt 0
template <typename T>
__global__ void bin_rows_kernel(const T* __restrict__ work, uint32_t rows, uint32_t s_max,
                                uint32_t m_max, uint32_t* __restrict__ lists,
                                uint32_t* __restrict__ counters, uint32_t* __restrict__ cnt_zero) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const uint64_t w = (uint64_t)work[r];
    if (w == 0) {
        if (cnt_zero) cnt_zero[r] = 0;
        return;
    }
    const int bin = w <= s_max ? 0 : (w <= m_max ? 1 : 2);
    const uint32_t pos = atomicAdd(&counters[bin], 1u);
    lists[(uint64_t)bin * rows + pos] = r;
}

// ---- symbolic, small rows: warp per row, 8-lane groups each take one A non-zero ---
__global__ void __launch_bounds__(NT)
    sym_small_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                     const uint32_t* __restrict__ b_ip, const uint32_t* __restrict__ b_idx,
                     const uint32_t* __restrict__ list, uint32_t n_list,
                     uint32_t* __restrict__ cnt) {
    __shared__ uint32_t tab[WARPS][S_SLOTS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = lane >> 3, gl = lane & 7;
    uint32_t* t = tab[warp];
    for (uint32_t li = blockIdx.x * WARPS + warp; li < n_list; li += gridDim.x * WARPS) {
        const uint32_t r = list[li];
        for (int i = lane; i < S_SLOTS; i += 32) t[i] = EMPTY;
        __syncwarp();
        uint32_t mine = 0;
        for (uint32_t k = a_ip[r] + grp, e = a_ip[r + 1]; k < e; k += 4) {
            const uint32_t br = a_idx[k];
            for (uint32_t p = b_ip[br] + gl, pe = b_ip[br + 1]; p < pe; p += 8) {
                bool fresh;
                table_insert(t, S_SLOTS - 1, b_idx[p], &fresh);
                mine += fresh;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
        if (lane == 0) cnt[r] = mine;
        __syncwarp();
    }
}

// ---- symbolic, medium rows: CTA per row, hash set in dynamic shared memory ---------
__global__ void __launch_bounds__(NT)
    sym_med_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                   const uint32_t* __restrict__ b_ip, const uint32_t* __restrict__ b_idx,
                   const uint64_t* __restrict__ nprod, const uint32_t* __restrict__ list,
                   uint32_t n_list, uint32_t* __restrict__ cnt, int grouping) {
    extern __shared__ uint32_t dyn_u32[];
    uint32_t* t = dyn_u32;
    __shared__ uint32_t total;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t li = blockIdx.x; li < n_list; li += gridDim.x) {
        const uint32_t r = list[li];
        uint32_t slots = 512;
        while (slots < 2 * (uint32_t)nprod[r]) slots <<= 1;  // <= SYM_M_SLOTS by binning
        for (uint32_t i = threadIdx.x; i < slots; i += NT) t[i] = EMPTY;
        if (threadIdx.x == 0) total = 0;
        __syncthreads();
        uint32_t mine = 0;
        const uint32_t a0 = a_ip[r], a1 = a_ip[r + 1];
        const int G = warps_per_brow(a1 - a0, WARPS, grouping);
        const int grp = warp / G, wg = warp % G, ngrp = WARPS / G;
        for (uint32_t k = a0 + grp; k < a1; k += ngrp) {
            const uint32_t br = a_idx[k];
            for (uint32_t p = b_ip[br] + wg * 32 + lane, pe = b_ip[br + 1]; p < pe; p += 32 * G) {
                bool fresh;
                table_insert(t, slots - 1, b_idx[p], &fresh);
                mine += fresh;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
        if (lane == 0 && mine) atomicAdd(&total, mine);
        __syncthreads();
        if (threadIdx.x == 0) cnt[r] = total;
        __syncthreads();
    }
}

// ---- symbolic, large rows: CTA per row, dense bitmap (shared or global slot) -------
// SMEM_BM: the bitmap's address space is a template parameter, not a run-time pointer choice
// (with the choice at run time the compiler has to emit generic ATOM.E.OR instead of ATOMS.OR
// for the shared-memory bitmap; cuobjdump of the first version).
constexpr int SYM_L_NT = 1024;  // one CTA per SM (the bitmap takes the shared memory)
template <bool SMEM_BM>
__global__ void __launch_bounds__(SYM_L_NT)
    sym_large_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                     const uint32_t* __restrict__ b_ip, const uint32_t* __restrict__ b_idx,
                     const uint32_t* __restrict__ list, uint32_t n_list, uint32_t words,
                     uint32_t* __restrict__ g_bitmaps /* used when !SMEM_BM */,
                     uint32_t* __restrict__ cnt, int grouping, uint32_t* __restrict__ row_counter) {
    constexpr int NTH = SYM_L_NT, NW = NTH / 32;
    extern __shared__ uint32_t dyn_u32[];
    uint32_t* bm = SMEM_BM ? dyn_u32 : g_bitmaps + (uint64_t)blockIdx.x * words;
    __shared__ uint32_t total;
    __shared__ uint32_t next_li;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t i = threadIdx.x; i < words; i += NTH) bm[i] = 0;  // re-zeroed by the count pass
    for (;;) {
        // rows are handed out dynamically: work per row spans three orders of magnitude
        if (threadIdx.x == 0) {
            next_li = atomicAdd(row_counter, 1u);
            total = 0;
        }
        __syncthreads();
        const uint32_t li = next_li;
        if (li >= n_list) break;
        const uint32_t r = list[li];
        const uint32_t a0 = a_ip[r], a1 = a_ip[r + 1];
        const int G = warps_per_brow(a1 - a0, NW, grouping);
        const int grp = warp / G, wg = warp % G, ngrp = NW / G;
        // the row range of the NEXT A non-zero is fetched while the current B row streams
        uint32_t k = a0 + grp, s = 0, e = 0;
        if (k < a1) {
            const uint32_t br = a_idx[k];
            s = b_ip[br];
            e = b_ip[br + 1];
        }
        while (k < a1) {
            const uint32_t kn = k + ngrp;
            uint32_t sn = 0, en = 0;
            if (kn < a1) {
                const uint32_t brn = a_idx[kn];
                sn = b_ip[brn];
                en = b_ip[brn + 1];
            }
            for (uint32_t p = s + (uint32_t)wg * 128 + lane; p < e; p += 128u * G) {
                uint32_t c[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) c[u] = (p + 32 * u < e) ? b_idx[p + 32 * u] : EMPTY;
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (c[u] != EMPTY) atomicOr(&bm[c[u] >> 5], 1u << (c[u] & 31));
            }
            k = kn;
            s = sn;
            e = en;
        }
        __syncthreads();
        uint32_t mine = 0;
        for (uint32_t i = threadIdx.x; i < words; i += NTH) {
            mine += __popc(bm[i]);
            bm[i] = 0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
        if (lane == 0 && mine) atomicAdd(&total, mine);
        __syncthreads();
        if (threadIdx.x == 0) cnt[r] = total;
        // next_li / total are rewritten only after the barrier at the top of the loop... which
        // thread 0 reaches after this store; the other threads read next_li before it
        __syncthreads();
    }
}

// ---- numeric, small rows: warp per row, sequential over A's non-zeros -> the exact
// summation order of smmp.rs:173-181 (bit-identical values) -----------------------
__global__ void __launch_bounds__(NT)
    num_small_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                     const double* __restrict__ a_val, const uint32_t* __restrict__ b_ip,
                     const uint32_t* __restrict__ b_idx, const double* __restrict__ b_val,
                     const uint64_t* __restrict__ c_ip, const uint32_t* __restrict__ list,
                     uint32_t n_list, uint32_t* __restrict__ c_idx, double* __restrict__ c_val) {
    __shared__ uint32_t tkey[WARPS][S_SLOTS];
    __shared__ double tval[WARPS][S_SLOTS];
    __shared__ uint32_t ckey[WARPS][NUM_S_MAX];
    __shared__ double cval[WARPS][NUM_S_MAX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* tk = tkey[warp];
    double* tv = tval[warp];
    for (uint32_t li = blockIdx.x * WARPS + warp; li < n_list; li += gridDim.x * WARPS) {
        const uint32_t r = list[li];
        for (int i = lane; i < S_SLOTS; i += 32) {
            tk[i] = EMPTY;
            tv[i] = 0.0;
        }
        __syncwarp();
        for (uint32_t k = a_ip[r], e = a_ip[r + 1]; k < e; ++k) {  // storage order
            const uint32_t br = a_idx[k];
            const double av = a_val[k];
            for (uint32_t p = b_ip[br] + lane, pe = b_ip[br + 1]; p < pe; p += 32) {
                bool fresh;
                const uint32_t slot = table_insert(tk, S_SLOTS - 1, b_idx[p], &fresh);
                // columns of one B row are distinct: no two lanes share a slot here
                tv[slot] = __dadd_rn(tv[slot], __dmul_rn(av, b_val[p]));
            }
            __syncwarp();
        }
        // compact, rank-sort by column, write
        uint32_t n = 0;
        for (int base = 0; base < S_SLOTS; base += 32) {
            const uint32_t key = tk[base + lane];
            const uint32_t m = __ballot_sync(0xffffffffu, key != EMPTY);
            if (key != EMPTY) {
                const uint32_t o = n + __popc(m & ((1u << lane) - 1u));
                ckey[warp][o] = key;
                cval[warp][o] = tv[base + lane];
            }
            n += __popc(m);
        }
        __syncwarp();
        const uint64_t out0 = c_ip[r];
        for (uint32_t i = lane; i < n; i += 32) {
            const uint32_t key = ckey[warp][i];
            uint32_t rank = 0;
            for (uint32_t j = 0; j < n; ++j) rank += ckey[warp][j] < key;
            c_idx[out0 + rank] = key;
            c_val[out0 + rank] = cval[warp][i];
        }
        __syncwarp();
    }
}

// ---- ordered accumulation for the CTA-per-row numeric kernels --------------------------
// The reference adds a row's products into tmp[j] one A non-zero after the other, in storage
// order, each sum starting from +0.0 (smmp.rs:173-181).  The CTA-per-row kernels keep that order
// under any thread schedule without floating-point atomics: a CTA takes the row's A non-zeros in
// rounds of one per warp, in storage order.  Each warp loads the first chunk (<= 32 products) of
// its B-row segment and stages (slot, product) at its place in the round's stream, so the staged
// list is in storage order; warp 0 then folds it into the accumulator.  A segment longer than one
// chunk ("long") is finished by the whole CTA in turn, right after the staged products before it:
// the products of one A non-zero have distinct columns, so its chunks need no order among
// themselves.  `ACC_GLOBAL` bypasses L1 for an accumulator in global memory.
template <bool ACC_GLOBAL>
__device__ __forceinline__ double acc_load(const double* p) {
    if constexpr (ACC_GLOBAL) return __ldcg(p);
    else return *p;
}
template <bool ACC_GLOBAL>
__device__ __forceinline__ void acc_store(double* p, double v) {
    if constexpr (ACC_GLOBAL) __stcg(p, v);
    else *p = v;
}

// warp 0: fold staged entries [s, e) into acc in stream order.  Lanes take 32 entries at a time;
// equal slots are grouped with match_any and the group's lowest lane adds the members in lane
// (= stream) order into the running value.
template <bool ACC_GLOBAL, typename S>
__device__ __forceinline__ void fold_staged(const S* st_slot, const double* st_val, uint32_t s,
                                            uint32_t e, double* acc, int lane) {
    for (uint32_t i = s; i < e; i += 32) {
        const uint32_t j = i + lane;
        const uint32_t slot = j < e ? (uint32_t)st_slot[j] : EMPTY;
        const uint32_t grp = __match_any_sync(0xffffffffu, slot);
        if (slot != EMPTY && (grp & ((1u << lane) - 1u)) == 0) {
            double sum = acc_load<ACC_GLOBAL>(acc + slot);
            for (uint32_t m = grp; m; m &= m - 1) sum = __dadd_rn(sum, st_val[i + __ffs(m) - 1]);
            acc_store<ACC_GLOBAL>(acc + slot, sum);
        }
        __syncwarp();
    }
}

// Per-round bookkeeping in shared memory for kernels whose segments are whole B rows (their
// length is known up front): chunk counts, and for long segments the rest of the B row.
struct RoundState {
    uint32_t cnt[32];   // products staged by each warp
    uint32_t rest0[32];  // long segments: first B position after the staged chunk
    uint32_t rest1[32];  // long segments: end of the B row
    double av[32];       // long segments: A's value
};

// One round of the ordered accumulation over whole B rows, A non-zeros [k0, k0 + nwarps).
// `slot_of(col)` maps a column to its accumulator slot (order-free: a hash insert or the
// column itself), `mark(col)` records the column for extraction.
template <bool ACC_GLOBAL, typename SlotOf, typename Mark>
__device__ __forceinline__ void ordered_round(
    const uint32_t* __restrict__ a_idx, const double* __restrict__ a_val,
    const uint32_t* __restrict__ b_ip, const uint32_t* __restrict__ b_idx,
    const double* __restrict__ b_val, uint32_t k0, uint32_t a1, double* acc,
    uint32_t* st_slot, double* st_val, RoundState& rs, SlotOf slot_of, Mark mark) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const uint32_t k = k0 + warp;
    uint32_t s = 0, len = 0;
    double av = 0.0;
    if (k < a1) {
        const uint32_t br = a_idx[k];
        s = b_ip[br];
        len = b_ip[br + 1] - s;
        av = a_val[k];
    }
    const uint32_t n = len < 32 ? len : 32;
    uint32_t slot = EMPTY;
    double prod = 0.0;
    if ((uint32_t)lane < n) {
        const uint32_t c = b_idx[s + lane];
        prod = __dmul_rn(av, b_val[s + lane]);
        slot = slot_of(c);
        mark(c);
    }
    if (lane == 0) {
        rs.cnt[warp] = n | (len > 32 ? 0x80000000u : 0u);
        rs.rest0[warp] = s + 32;
        rs.rest1[warp] = s + len;
        rs.av[warp] = av;
    }
    __syncthreads();
    // exclusive offsets of the warps' chunks in the round's stream (every warp computes them)
    const uint32_t wc = lane < nwarps ? rs.cnt[lane] : 0u;
    const uint32_t longs = __ballot_sync(0xffffffffu, wc >> 31);
    uint32_t incl = wc & 0x7fffffffu;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    const uint32_t off = __shfl_sync(0xffffffffu, incl, warp) - n;
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    if ((uint32_t)lane < n) {
        st_slot[off + lane] = slot;
        st_val[off + lane] = prod;
    }
    __syncthreads();
    uint32_t from = 0;
    for (uint32_t lm = longs; lm; lm &= lm - 1) {  // uniform
        const int L = __ffs(lm) - 1;
        const uint32_t upto = __shfl_sync(0xffffffffu, incl, L);
        if (warp == 0) fold_staged<ACC_GLOBAL>(st_slot, st_val, from, upto, acc, lane);
        __syncthreads();
        const double lav = rs.av[L];
        for (uint32_t p = rs.rest0[L] + threadIdx.x, e = rs.rest1[L]; p < e; p += blockDim.x) {
            const uint32_t c = b_idx[p];
            const uint32_t sl = slot_of(c);
            mark(c);
            acc_store<ACC_GLOBAL>(acc + sl, __dadd_rn(acc_load<ACC_GLOBAL>(acc + sl),
                                                      __dmul_rn(lav, b_val[p])));
        }
        __syncthreads();
        from = upto;
    }
    if (warp == 0) fold_staged<ACC_GLOBAL>(st_slot, st_val, from, total, acc, lane);
    // the next round writes the stage only after its first barrier, which warp 0 reaches once
    // its fold is done; `rs` is read above before the second barrier of this round
}

// ---- numeric, medium rows: CTA per row, hash map in shared memory + bitonic sort ----
__global__ void __launch_bounds__(NT)
    num_med_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                   const double* __restrict__ a_val, const uint32_t* __restrict__ b_ip,
                   const uint32_t* __restrict__ b_idx, const double* __restrict__ b_val,
                   const uint64_t* __restrict__ c_ip, const uint32_t* __restrict__ cnt,
                   const uint32_t* __restrict__ list, uint32_t n_list,
                   uint32_t* __restrict__ c_idx, double* __restrict__ c_val) {
    extern __shared__ __align__(16) unsigned char dyn_raw[];
    double* tv = (double*)dyn_raw;                               // NUM_M_SLOTS doubles
    uint32_t* tk = (uint32_t*)(dyn_raw + NUM_M_SLOTS * sizeof(double));
    __shared__ uint32_t st_slot[NT];
    __shared__ double st_val[NT];
    __shared__ RoundState rs;
    for (uint32_t li = blockIdx.x; li < n_list; li += gridDim.x) {
        const uint32_t r = list[li];
        const uint32_t n = cnt[r];
        uint32_t slots = 512;
        while (slots < 2 * n) slots <<= 1;
        for (uint32_t i = threadIdx.x; i < slots; i += NT) {
            tk[i] = EMPTY;
            tv[i] = 0.0;
        }
        __syncthreads();
        const uint32_t a0 = a_ip[r], a1 = a_ip[r + 1];
        auto slot_of = [&](uint32_t c) {
            bool fresh;
            return table_insert(tk, slots - 1, c, &fresh);
        };
        auto mark = [](uint32_t) {};
        for (uint32_t k0 = a0; k0 < a1; k0 += WARPS)
            ordered_round<false>(a_idx, a_val, b_ip, b_idx, b_val, k0, a1, tv, st_slot, st_val, rs,
                                 slot_of, mark);
        __syncthreads();
        // in-place bitonic sort of (key, val) by key; EMPTY = +inf sinks to the end
        for (uint32_t size = 2; size <= slots; size <<= 1) {
            for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
                for (uint32_t i = threadIdx.x; i < (slots >> 1); i += NT) {
                    const uint32_t lo = 2 * i - (i & (stride - 1));
                    const uint32_t hi = lo + stride;
                    const bool up = (lo & size) == 0;
                    const uint32_t kl = tk[lo], kh = tk[hi];
                    if ((kl > kh) == up) {
                        tk[lo] = kh;
                        tk[hi] = kl;
                        const double t = tv[lo];
                        tv[lo] = tv[hi];
                        tv[hi] = t;
                    }
                }
                __syncthreads();
            }
        }
        const uint64_t out0 = c_ip[r];
        for (uint32_t i = threadIdx.x; i < n; i += NT) {
            c_idx[out0 + i] = tk[i];
            c_val[out0 + i] = tv[i];
        }
        __syncthreads();
    }
}

// ---- numeric, large rows: dense accumulator slot in global memory + bitmap --------
template <bool SMEM_BM>
__global__ void __launch_bounds__(1024)
    num_large_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                     const double* __restrict__ a_val, const uint32_t* __restrict__ b_ip,
                     const uint32_t* __restrict__ b_idx, const double* __restrict__ b_val,
                     const uint64_t* __restrict__ c_ip, const uint32_t* __restrict__ list,
                     uint32_t n_list, uint32_t words, uint64_t cols,
                     uint32_t* __restrict__ g_bitmaps /* used when !SMEM_BM */,
                     double* __restrict__ g_acc /* gridDim.x * cols, zero on entry */,
                     uint32_t* __restrict__ c_idx, double* __restrict__ c_val) {
    extern __shared__ uint32_t dyn_u32[];
    uint32_t* bm = SMEM_BM ? dyn_u32 : g_bitmaps + (uint64_t)blockIdx.x * words;
    double* acc = g_acc + (uint64_t)blockIdx.x * cols;
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t chunk_total;
    __shared__ uint32_t st_slot[1024];
    __shared__ double st_val[1024];
    __shared__ RoundState rs;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nt = blockDim.x, nwarps = blockDim.x >> 5;  // 256..1024 threads
    for (uint32_t li = blockIdx.x; li < n_list; li += gridDim.x) {
        const uint32_t r = list[li];
        for (uint32_t i = threadIdx.x; i < words; i += nt) bm[i] = 0;
        __syncthreads();
        auto slot_of = [](uint32_t c) { return c; };
        auto mark = [&](uint32_t c) { atomicOr(&bm[c >> 5], 1u << (c & 31)); };
        for (uint32_t k0 = a_ip[r], a1 = a_ip[r + 1]; k0 < a1; k0 += nwarps)
            ordered_round<true>(a_idx, a_val, b_ip, b_idx, b_val, k0, a1, acc, st_slot, st_val, rs,
                                slot_of, mark);
        __syncthreads();
        // ordered extraction: walk the bitmap 256 words at a time
        uint64_t out = c_ip[r];
        for (uint32_t w0 = 0; w0 < words; w0 += nt) {
            const uint32_t w = w0 + threadIdx.x;
            uint32_t bits = w < words ? bm[w] : 0u;
            const uint32_t c = __popc(bits);
            uint32_t inc = c;  // block exclusive scan of c
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += u;
            }
            if (lane == 31) wsum[warp] = inc;
            __syncthreads();
            if (warp == 0) {
                uint32_t v = lane < (int)nwarps ? wsum[lane] : 0u, vi = v;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(0xffffffffu, vi, o);
                    if (lane >= o) vi += u;
                }
                wsum[lane] = vi - v;
                if (lane == 31) chunk_total = vi;
            }
            __syncthreads();
            uint64_t o = out + wsum[warp] + inc - c;
            while (bits) {
                const uint32_t b = __ffs(bits) - 1;
                bits &= bits - 1;
                const uint32_t col = w * 32 + b;
                c_idx[o] = col;
                c_val[o] = __ldcg(&acc[col]);
                __stcg(&acc[col], 0.0);  // leave the slot zeroed for the next row
                ++o;
            }
            out += chunk_total;
            __syncthreads();
        }
    }
}

// ---- numeric, large rows with a moderate A row (<= PANEL_MAX_A non-zeros): dense f64
// accumulation in SHARED memory, one column panel of PANEL_W columns at a time.  Per A
// non-zero a cursor remembers how far its (sorted) B row has been consumed, so every B entry is
// read once and lands in the panel that owns its column; panels are extracted in order, so the
// row comes out sorted.  No global atomics (round 1's dense accumulators in global memory were
// 77 % of the whole SpGEMM).  Everything a segment needs -- cursor, end of the B row, A's value
// -- sits in shared memory (filled once per row): one dependent global load per chunk instead of
// three; 1024 threads, rows handed out dynamically, panels nothing landed in are skipped.  The
// products are added in the reference's order (see ordered_round): the round's stage keeps
// 16-bit panel columns, so it fits beside the 210 KB below without shrinking PANEL_W or
// PANEL_MAX_A.  On config 4 nearly every product comes from a B row longer than one chunk,
// and each such segment costs the CTA a turn (two barriers, one L2 round trip): this kernel
// takes 2.3x the time of the former arrival-order version there (DESIGN.md §11).
constexpr uint32_t PANEL_W = 16384;       // columns per panel: 128 KB of f64 accumulators
constexpr uint32_t PANEL_MAX_A = 4096;    // per-A-non-zero state: 16 B each = 64 KB
constexpr size_t PANEL_SMEM = (size_t)PANEL_W * 8 + PANEL_W / 8 + (size_t)PANEL_MAX_A * 20;
constexpr int PANEL_NT = 1024;

__global__ void __launch_bounds__(PANEL_NT)
    num_panel_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ a_idx,
                     const double* __restrict__ a_val, const uint32_t* __restrict__ b_ip,
                     const uint32_t* __restrict__ b_idx, const double* __restrict__ b_val,
                     const uint64_t* __restrict__ c_ip, const uint32_t* __restrict__ list,
                     uint32_t n_list, uint32_t cols, uint32_t* __restrict__ c_idx,
                     double* __restrict__ c_val, uint32_t* __restrict__ row_counter) {
    constexpr int NTH = PANEL_NT, NWARPS = NTH / 32;
    extern __shared__ __align__(16) unsigned char dyn_raw[];
    double* acc = (double*)dyn_raw;                                  // PANEL_W
    double* aval = acc + PANEL_W;                                     // PANEL_MAX_A
    uint32_t* bm = (uint32_t*)(aval + PANEL_MAX_A);                   // PANEL_W / 32 words
    uint32_t* cursor = bm + PANEL_W / 32;                             // PANEL_MAX_A
    uint32_t* bend = cursor + PANEL_MAX_A;                            // PANEL_MAX_A
    uint32_t* nextcol = bend + PANEL_MAX_A;  // column at the cursor (0 = not known yet): a B row
                                             // with nothing in a panel costs one LDS there
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t chunk_total;
    __shared__ uint32_t panel_mark;  // sequence number of the last panel something landed in
    __shared__ uint32_t next_li;
    // the round's stage (16-bit panel columns keep it beside the 210 KB above) and, per warp,
    // its chunk count (bit 31: long), its A non-zero and a long segment's rest, end and A value
    __shared__ uint16_t st_slot[NTH];
    __shared__ double st_val[NTH];
    __shared__ uint32_t lcnt[NWARPS], lkk[NWARPS], lrest[NWARPS], lend[NWARPS];
    __shared__ double lav[NWARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t i = threadIdx.x; i < PANEL_W; i += NTH) acc[i] = 0.0;   // stays zero between rows
    for (uint32_t i = threadIdx.x; i < PANEL_W / 32; i += NTH) bm[i] = 0;
    if (threadIdx.x == 0) panel_mark = 0;
    __syncthreads();
    uint32_t seq = 0;  // panels visited by this CTA so far (uniform)
    for (;;) {
        if (threadIdx.x == 0) next_li = atomicAdd(row_counter, 1u);
        __syncthreads();
        const uint32_t li = next_li;  // the next write is behind the barrier after the set-up
        if (li >= n_list) break;
        const uint32_t r = list[li];
        const uint32_t a0 = a_ip[r], na = a_ip[r + 1] - a0;
        for (uint32_t kk = threadIdx.x; kk < na; kk += NTH) {
            const uint32_t br = a_idx[a0 + kk];
            cursor[kk] = b_ip[br];
            bend[kk] = b_ip[br + 1];
            aval[kk] = a_val[a0 + kk];
            nextcol[kk] = 0;
        }
        __syncthreads();
        uint64_t out = c_ip[r];
        for (uint32_t p0 = 0; p0 < cols; p0 += PANEL_W) {
            const uint32_t p1 = (cols - p0 > PANEL_W) ? p0 + PANEL_W : cols;
            ++seq;
            // ordered accumulation (see ordered_round): rounds of one A non-zero per warp; the
            // segment of A non-zero kk in this panel is the prefix of [cursor, end) below p1
            // (columns ascend), its first chunk is staged, a longer one is finished by the CTA
            for (uint32_t k0 = 0; k0 < na; k0 += NWARPS) {
                // (the first column beyond the cursor is known from the last visit, 0 = unknown)
                const uint32_t kk = k0 + warp < na && nextcol[k0 + warp] < p1 ? k0 + warp : EMPTY;
                uint32_t n = 0, pos = 0, end = 0, c = EMPTY;
                bool lng = false;
                double av = 0.0, v = 0.0;
                uint32_t nxt = 0;
                if (kk != EMPTY) {
                    pos = cursor[kk];
                    end = bend[kk];
                    av = aval[kk];
                    if (pos + lane < end) {
                        c = b_idx[pos + lane];
                        v = b_val[pos + lane];
                    }
                    n = __popc(__ballot_sync(0xffffffffu, c < p1));
                    lng = n == 32 && pos + 32 < end;
                    const uint32_t nc = __shfl_sync(0xffffffffu, c, n & 31);
                    nxt = lng ? 0u : (n < 32 ? nc : EMPTY);  // EMPTY: row used up
                    if (lane == 0 && n) panel_mark = seq;     // same value from every writer
                }
                if (lane == 0) {
                    lcnt[warp] = n | (lng ? 0x80000000u : 0u);
                    lkk[warp] = kk;
                    lrest[warp] = pos + 32;
                    lend[warp] = end;
                    lav[warp] = av;
                }
                __syncthreads();
                if (kk != EMPTY && lane == 0) {
                    cursor[kk] = pos + n;  // a long segment adds its rest below
                    nextcol[kk] = nxt;
                }
                const uint32_t wc = lane < NWARPS ? lcnt[lane] : 0u;
                const uint32_t longs = __ballot_sync(0xffffffffu, wc >> 31);
                uint32_t incl = wc & 0x7fffffffu;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += u;
                }
                const uint32_t off = __shfl_sync(0xffffffffu, incl, warp) - n;
                const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
                if ((uint32_t)lane < n) {
                    st_slot[off + lane] = (uint16_t)(c - p0);
                    st_val[off + lane] = __dmul_rn(av, v);
                    atomicOr(&bm[(c - p0) >> 5], 1u << ((c - p0) & 31));
                }
                __syncthreads();
                uint32_t from = 0;
                for (uint32_t lm = longs; lm; lm &= lm - 1) {  // uniform
                    const int L = __ffs(lm) - 1;
                    const uint32_t upto = __shfl_sync(0xffffffffu, incl, L);
                    if (warp == 0) fold_staged<false>(st_slot, st_val, from, upto, acc, lane);
                    __syncthreads();
                    // the taken entries are a prefix: each warp stops at its first partial chunk
                    const uint32_t q0 = lrest[L], e = lend[L];
                    const double lv = lav[L];
                    uint32_t mine = 0;
                    for (uint32_t q = q0 + warp * 32u; q < e; q += NWARPS * 32u) {
                        const uint32_t p = q + lane;
                        const uint32_t cl = p < e ? b_idx[p] : EMPTY;
                        const bool take = cl < p1;
                        if (take) {
                            acc[cl - p0] = __dadd_rn(acc[cl - p0], __dmul_rn(lv, b_val[p]));
                            atomicOr(&bm[(cl - p0) >> 5], 1u << ((cl - p0) & 31));
                        }
                        const uint32_t nn = __popc(__ballot_sync(0xffffffffu, take));
                        mine += nn;
                        if (nn < 32) break;
                    }
                    if (lane == 0 && mine) atomicAdd(&cursor[lkk[L]], mine);
                    __syncthreads();
                    from = upto;
                }
                if (warp == 0) fold_staged<false>(st_slot, st_val, from, total, acc, lane);
            }
            __syncthreads();
            if (panel_mark != seq) {  // nothing landed here (uniform: read after the barrier)
                __syncthreads();      // cursor updates above / panel_mark before the next panel
                continue;
            }
            // ordered extraction of this panel (also re-zeroes what it touched)
            const uint32_t words = (p1 - p0 + 31) / 32;
            for (uint32_t w0 = 0; w0 < words; w0 += NTH) {
                const uint32_t w = w0 + threadIdx.x;
                uint32_t bits = w < words ? bm[w] : 0u;
                if (w < words) bm[w] = 0;
                const uint32_t c = __popc(bits);
                uint32_t inc = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
                    if (lane >= o) inc += u;
                }
                if (lane == 31) wsum[warp] = inc;
                __syncthreads();
                if (warp == 0) {
                    uint32_t v = lane < NWARPS ? wsum[lane] : 0u, vi = v;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t u = __shfl_up_sync(0xffffffffu, vi, o);
                        if (lane >= o) vi += u;
                    }
                    wsum[lane] = vi - v;
                    if (lane == 31) chunk_total = vi;
                }
                __syncthreads();
                uint64_t o = out + wsum[warp] + inc - c;
                while (bits) {
                    const uint32_t b = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const uint32_t lc = w * 32 + b;
                    c_idx[o] = p0 + lc;
                    c_val[o] = acc[lc];
                    acc[lc] = 0.0;
                    ++o;
                }
                out += chunk_total;
                __syncthreads();
            }
        }
    }
}

template <typename TIn, typename TOut>
__global__ void widen_kernel(const TIn* __restrict__ in, TOut* __restrict__ out, uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = (TOut)in[i];
}

// split the numeric "large" list by the length of the A row: short A rows -> panel kernel
__global__ void split_large_kernel(const uint32_t* __restrict__ a_ip, const uint32_t* __restrict__ list,
                                   uint32_t n_list, uint32_t max_a, uint32_t* __restrict__ panel_list,
                                   uint32_t* __restrict__ hub_list, uint32_t* __restrict__ counters) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_list) return;
    const uint32_t r = list[i];
    const bool hub = a_ip[r + 1] - a_ip[r] > max_a;
    const uint32_t pos = atomicAdd(&counters[hub ? 4 : 3], 1u);
    (hub ? hub_list : panel_list)[pos] = r;
}

inline unsigned grid_for(uint64_t n) { return (unsigned)((n + 255) / 256); }

int check_operands(sprs_b200_ctx* ctx, const sprs_b200_csmat* a, const sprs_b200_csmat* b) {
    // the reference asserts lhs.cols() == rhs.rows() first (smmp.rs:207)
    if (a->cols != b->rows) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (a->storage != SPRS_B200_CSR || b->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch");
    if (a->indptr_bytes != 4 || b->indptr_bytes != 4)
        SPRS_FAIL(ctx, SPRS_B200_ERR_UNSUPPORTED, "spgemm operands need nnz < 2^32");
    return SPRS_B200_OK;
}

struct LargeWorkspace {
    uint32_t* bitmaps = nullptr;
    double* acc = nullptr;
    unsigned grid = 0;
    size_t smem = 0;
    uint32_t words = 0;
};

void free_large(LargeWorkspace& w) {
    if (w.bitmaps) cudaFree(w.bitmaps);
    if (w.acc) cudaFree(w.acc);
    w.bitmaps = nullptr;
    w.acc = nullptr;
}

// bitmap placement (+ dense accumulators when need_acc) for the large-row kernels
int plan_large(sprs_b200_ctx* ctx, uint64_t cols, uint32_t n_large, bool need_acc,
               LargeWorkspace* w, cudaStream_t s) {
    w->words = (uint32_t)((cols + 31) / 32);
    unsigned grid = (unsigned)std::min<uint64_t>(n_large, (uint64_t)ctx->sm_count * 2);
    if (need_acc) {  // bound the dense slots to ~8 GB (10 % of an H100's 80 GB)
        const uint64_t per = cols * sizeof(double);
        const uint64_t cap = std::max<uint64_t>(1, (8ull << 30) / std::max<uint64_t>(per, 1));
        grid = (unsigned)std::min<uint64_t>(grid, cap);
    }
    if (grid == 0) grid = 1;
    w->grid = grid;
    const bool smem_bitmap = cols <= BITMAP_SMEM_MAX_COLS;
    w->smem = smem_bitmap ? (size_t)w->words * 4 : 0;
    if (!smem_bitmap)
        SPRS_CUDA(ctx, cudaMalloc((void**)&w->bitmaps, (size_t)grid * w->words * 4));
    if (need_acc) {
        SPRS_CUDA(ctx, cudaMalloc((void**)&w->acc, (size_t)grid * cols * sizeof(double)));
        SPRS_CUDA(ctx, cudaMemsetAsync(w->acc, 0, (size_t)grid * cols * sizeof(double), s));
    }
    return SPRS_B200_OK;
}

int run_numeric(sprs_b200_ctx* ctx, sprs_b200_spgemm* p, uint32_t* d_cidx, double* d_cval,
                cudaStream_t s) {
    if (p->rows == 0 || p->nnz_c == 0) return SPRS_B200_OK;
    const uint32_t rows = (uint32_t)p->rows;
    const auto* a = p->a;
    const auto* b = p->b;
    const uint32_t *a_ip = (const uint32_t*)a->d_indptr, *b_ip = (const uint32_t*)b->d_indptr;
    SPRS_CUDA(ctx, cudaMemsetAsync(p->d_counters, 0, 8 * sizeof(uint32_t), s));
    // rows with more than 16 entries per column panel are cheaper in the panel kernel (no
    // probing, no sort; fixed cost ~ n_panels) than in the CTA hash map
    // Hash map or panels?  A row costs the panel kernel ~900 instructions per warp and panel
    // whatever it holds, the CTA hash map pays per product plus a bitonic sort of its table:
    // the cut sits at 1024 entries.
    const uint32_t num_m_max = std::min<uint32_t>(NUM_M_MAX, 1024);
    bin_rows_kernel<uint32_t><<<grid_for(rows), 256, 0, s>>>(p->d_cnt, rows, NUM_S_MAX, num_m_max,
                                                            p->d_lists, p->d_counters, nullptr);
    ctx->launches += 1;
    uint32_t h_cnt[8];
    SPRS_CUDA(ctx, cudaMemcpyAsync(h_cnt, p->d_counters, sizeof(h_cnt), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    const uint32_t *l0 = p->d_lists, *l1 = p->d_lists + rows, *l2 = p->d_lists + 2ull * rows;
    const unsigned cap = (unsigned)ctx->sm_count * 8;
    if (h_cnt[0]) {
        const unsigned g = std::min<unsigned>((h_cnt[0] + WARPS - 1) / WARPS, cap * 4);
        num_small_kernel<<<g, NT, 0, s>>>(a_ip, a->d_indices, a->d_data, b_ip, b->d_indices,
                                          b->d_data, p->d_cptr, l0, h_cnt[0], d_cidx, d_cval);
        ctx->launches += 1;
    }
    if (h_cnt[1]) {
        const size_t smem = NUM_M_SLOTS * (sizeof(double) + sizeof(uint32_t));
        SPRS_CUDA(ctx, cudaFuncSetAttribute(num_med_kernel,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const unsigned g = std::min<unsigned>(h_cnt[1], cap);
        num_med_kernel<<<g, NT, smem, s>>>(a_ip, a->d_indices, a->d_data, b_ip, b->d_indices,
                                           b->d_data, p->d_cptr, p->d_cnt, l1, h_cnt[1], d_cidx,
                                           d_cval);
        ctx->launches += 1;
    }
    if (h_cnt[2]) {
        // lists[0 .. rows) and [rows .. 2 rows) are free again once small / medium have been
        // LAUNCHED?  No -- they are still being read; use fresh scratch for the split lists.
        uint32_t* split = nullptr;
        SPRS_CUDA(ctx, cudaMallocAsync((void**)&split, 2ull * h_cnt[2] * sizeof(uint32_t), s));
        uint32_t *panel_list = split, *hub_list = split + h_cnt[2];
        split_large_kernel<<<grid_for(h_cnt[2]), 256, 0, s>>>(a_ip, l2, h_cnt[2], PANEL_MAX_A,
                                                             panel_list, hub_list, p->d_counters);
        ctx->launches += 1;
        uint32_t h2[8];
        cudaMemcpyAsync(h2, p->d_counters, sizeof(h2), cudaMemcpyDeviceToHost, s);
        int st = cudaStreamSynchronize(s) == cudaSuccess ? SPRS_B200_OK : SPRS_B200_ERR_CUDA;
        const uint32_t n_panel = h2[3], n_hub = h2[4];
        if (st == SPRS_B200_OK && n_panel) {
            auto kern = num_panel_kernel;
            if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)PANEL_SMEM) != cudaSuccess)
                st = SPRS_B200_ERR_CUDA;
            else {
                const unsigned g = std::min<unsigned>(n_panel, (unsigned)ctx->sm_count);
                kern<<<g, PANEL_NT, PANEL_SMEM, s>>>(a_ip, a->d_indices, a->d_data, b_ip,
                                                           b->d_indices, b->d_data, p->d_cptr,
                                                           panel_list, n_panel, (uint32_t)p->cols,
                                                           d_cidx, d_cval, p->d_counters + 5);
                ctx->launches += 1;
            }
        }
        if (st == SPRS_B200_OK && n_hub) {
            LargeWorkspace w;
            st = plan_large(ctx, p->cols, n_hub, true, &w, s);
            auto kern = w.smem ? num_large_kernel<true> : num_large_kernel<false>;
            if (st == SPRS_B200_OK && w.smem)
                if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)w.smem) != cudaSuccess)
                    st = SPRS_B200_ERR_CUDA;
            if (st == SPRS_B200_OK) {
                const unsigned big_nt = w.grid < (unsigned)ctx->sm_count ? 1024 : NT;
                kern<<<w.grid, big_nt, w.smem, s>>>(
                    a_ip, a->d_indices, a->d_data, b_ip, b->d_indices, b->d_data, p->d_cptr,
                    hub_list, n_hub, w.words, p->cols, w.bitmaps, w.acc, d_cidx, d_cval);
                ctx->launches += 1;
                if (cudaStreamSynchronize(s) != cudaSuccess) st = SPRS_B200_ERR_CUDA;
            }
            free_large(w);
        }
        if (cudaStreamSynchronize(s) != cudaSuccess) st = SPRS_B200_ERR_CUDA;
        cudaFreeAsync(split, s);
        if (st != SPRS_B200_OK) SPRS_FAIL(ctx, st, "spgemm numeric (large rows) failed");
    }
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

}  // namespace

extern "C" {

int sprs_b200_spgemm_symbolic(sprs_b200_ctx* ctx, const sprs_b200_csmat* a,
                              const sprs_b200_csmat* b, sprs_b200_spgemm** plan,
                              uint64_t* nnz_c) {
    if (!ctx || !a || !b || !plan || !nnz_c) return SPRS_B200_ERR_ARGUMENT;
    *plan = nullptr;
    *nnz_c = 0;
    SPRS_TRY(check_operands(ctx, a, b));
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    auto* p = new sprs_b200_spgemm();
    p->ctx = ctx;
    p->a = a;
    p->b = b;
    p->rows = a->rows;
    p->cols = b->cols;
    const uint32_t rows = (uint32_t)p->rows;
    int st = SPRS_B200_OK;
    do {
        // (stream-ordered allocations: the pool keeps the memory across calls, api.cu)
        if (cudaMallocAsync((void**)&p->d_nprod, (p->rows + 1) * 8, s) != cudaSuccess ||
            cudaMallocAsync((void**)&p->d_cnt, (p->rows + 1) * 4, s) != cudaSuccess ||
            cudaMallocAsync((void**)&p->d_cptr, (p->rows + 1) * 8, s) != cudaSuccess ||
            cudaMallocAsync((void**)&p->d_lists, (3 * p->rows + 1) * 4, s) != cudaSuccess ||
            cudaMallocAsync((void**)&p->d_counters, 8 * 4, s) != cudaSuccess) {
            sprs_b200_set_error(ctx, "spgemm: cudaMalloc failed");
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        cudaMemsetAsync(p->d_cptr, 0, (p->rows + 1) * 8, s);
        if (rows == 0) break;
        const uint32_t *a_ip = (const uint32_t*)a->d_indptr, *b_ip = (const uint32_t*)b->d_indptr;
        const unsigned cap = (unsigned)ctx->sm_count * 8;
        nprod_kernel<<<std::min<unsigned>((rows + WARPS - 1) / WARPS, cap * 4), NT, 0, s>>>(
            a_ip, a->d_indices, b_ip, rows, p->d_nprod);
        cudaMemsetAsync(p->d_counters, 0, 8 * sizeof(uint32_t), s);
            // with the bitmap in shared memory (no probing, fixed cost ~ cols / 32 words) the
        // hash set only pays below ~cols/256 products
        uint32_t sym_m_max = SYM_M_MAX;
        if (p->cols <= BITMAP_SMEM_MAX_COLS)
            sym_m_max = (uint32_t)std::min<uint64_t>(SYM_M_MAX, std::max<uint64_t>(SYM_S_MAX, p->cols / 256));
        bin_rows_kernel<uint64_t><<<grid_for(rows), 256, 0, s>>>(
            p->d_nprod, rows, SYM_S_MAX, sym_m_max, p->d_lists, p->d_counters, p->d_cnt);
        ctx->launches += 2;
        uint32_t h_cnt[8];
        if (cudaMemcpyAsync(h_cnt, p->d_counters, sizeof(h_cnt), cudaMemcpyDeviceToHost, s) !=
                cudaSuccess ||
            cudaStreamSynchronize(s) != cudaSuccess) {
            sprs_b200_set_error(ctx, "spgemm symbolic: binning failed");
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        const uint32_t *l0 = p->d_lists, *l1 = p->d_lists + rows, *l2 = p->d_lists + 2ull * rows;
        if (h_cnt[0]) {
            sym_small_kernel<<<std::min<unsigned>((h_cnt[0] + WARPS - 1) / WARPS, cap * 4), NT, 0,
                               s>>>(a_ip, a->d_indices, b_ip, b->d_indices, l0, h_cnt[0],
                                    p->d_cnt);
            ctx->launches += 1;
        }
        if (h_cnt[1]) {
            const size_t smem = SYM_M_SLOTS * sizeof(uint32_t);
            cudaFuncSetAttribute(sym_med_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem);
            sym_med_kernel<<<std::min<unsigned>(h_cnt[1], cap), NT, smem, s>>>(
                a_ip, a->d_indices, b_ip, b->d_indices, p->d_nprod, l1, h_cnt[1], p->d_cnt,
                1);
            ctx->launches += 1;
        }
        if (h_cnt[2]) {
            LargeWorkspace w;
            if ((st = plan_large(ctx, p->cols, h_cnt[2], false, &w, s)) != SPRS_B200_OK) break;
            auto kern = w.smem ? sym_large_kernel<true> : sym_large_kernel<false>;
            if (w.smem)
                cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)w.smem);
            kern<<<w.grid, SYM_L_NT, w.smem, s>>>(a_ip, a->d_indices, b_ip, b->d_indices, l2,
                                                  h_cnt[2], w.words, w.bitmaps, p->d_cnt, 1,
                                                  p->d_counters + 5);
            ctx->launches += 1;
            cudaStreamSynchronize(s);
            free_large(w);
        }
        if ((st = device_exclusive_scan<uint32_t, uint64_t>(ctx, p->d_cnt, rows, p->d_cptr, s)) !=
            SPRS_B200_OK)
            break;
        // n_prod total: scan of per-row n_prod would need another buffer; reduce on the host
        // side of the plan lazily (sprs_b200_spgemm_nprod)
        if (cudaMemcpyAsync(&p->nnz_c, p->d_cptr + rows, 8, cudaMemcpyDeviceToHost, s) !=
                cudaSuccess ||
            cudaStreamSynchronize(s) != cudaSuccess || cudaGetLastError() != cudaSuccess) {
            sprs_b200_set_error(ctx, "spgemm symbolic: kernel failed");
            st = SPRS_B200_ERR_CUDA;
        }
    } while (0);
    if (st != SPRS_B200_OK) {
        sprs_b200_spgemm_free(p);
        return st;
    }
    *plan = p;
    *nnz_c = p->nnz_c;
    return SPRS_B200_OK;
}

int sprs_b200_spgemm_numeric_dev(sprs_b200_ctx* ctx, sprs_b200_spgemm* p, sprs_b200_csmat** c) {
    if (!ctx || !p || !c) return SPRS_B200_ERR_ARGUMENT;
    *c = nullptr;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    auto* m = new sprs_b200_csmat();
    m->ctx = ctx;
    m->storage = SPRS_B200_CSR;
    m->rows = p->rows;
    m->cols = p->cols;
    m->nnz = p->nnz_c;
    m->outer = p->rows;
    m->inner = p->cols;
    m->indptr_bytes = p->nnz_c >= 0xffffffffull ? 8 : 4;
    m->pooled = true;
    int st = SPRS_B200_OK;
    do {
        if (cudaMallocAsync(&m->d_indptr, (m->rows + 1) * (size_t)m->indptr_bytes + 16, s) != cudaSuccess ||
            cudaMallocAsync((void**)&m->d_indices, m->nnz * 4 + 16, s) != cudaSuccess ||
            cudaMallocAsync((void**)&m->d_data, m->nnz * 8 + 16, s) != cudaSuccess) {
            sprs_b200_set_error(ctx, "spgemm numeric: cudaMalloc of C failed");
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        if (m->indptr_bytes == 4) {
            widen_kernel<uint64_t, uint32_t><<<grid_for(m->rows + 1), 256, 0, s>>>(
                p->d_cptr, (uint32_t*)m->d_indptr, m->rows + 1);
            ctx->launches += 1;
        } else {
            cudaMemcpyAsync(m->d_indptr, p->d_cptr, (m->rows + 1) * 8, cudaMemcpyDeviceToDevice, s);
        }
        if ((st = run_numeric(ctx, p, m->d_indices, m->d_data, s)) != SPRS_B200_OK) break;
        // (no SpMV hot set for a product: its build would run inside every SpGEMM call and
        // would need 4 more bytes per non-zero next to a result that may fill the device)
        if ((st = spmv_prepare(ctx, m, s, false)) != SPRS_B200_OK) break;
        if (cudaStreamSynchronize(s) != cudaSuccess || cudaGetLastError() != cudaSuccess) {
            sprs_b200_set_error(ctx, "spgemm numeric: kernel failed");
            st = SPRS_B200_ERR_CUDA;
        }
    } while (0);
    if (st != SPRS_B200_OK) {
        sprs_b200_csmat_free(m);
        return st;
    }
    *c = m;
    return SPRS_B200_OK;
}

int sprs_b200_spgemm_numeric(sprs_b200_ctx* ctx, sprs_b200_spgemm* p, void* c_indptr,
                             int indptr_bytes, void* c_indices, int index_bytes,
                             double* c_data) {
    if (!ctx || !p || !c_indptr) return SPRS_B200_ERR_ARGUMENT;
    if (p->nnz_c && (!c_indices || !c_data)) return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_csmat* c = nullptr;
    SPRS_TRY(sprs_b200_spgemm_numeric_dev(ctx, p, &c));
    const int st = sprs_b200_csmat_download(ctx, c, c_indptr, indptr_bytes, c_indices,
                                            index_bytes, c_data);
    sprs_b200_csmat_free(c);
    return st;
}

uint64_t sprs_b200_spgemm_nprod(const sprs_b200_spgemm* p) {
    if (!p || !p->d_nprod || p->rows == 0) return 0;
    auto* q = const_cast<sprs_b200_spgemm*>(p);
    if (q->n_prod == 0) {
        std::vector<uint64_t> h(p->rows);
        cudaSetDevice(p->ctx->device);
        if (cudaMemcpy(h.data(), p->d_nprod, p->rows * 8, cudaMemcpyDeviceToHost) == cudaSuccess)
            for (uint64_t v : h) q->n_prod += v;
    }
    return q->n_prod;
}

int sprs_b200_spgemm_free(sprs_b200_spgemm* p) {
    if (!p) return SPRS_B200_OK;
    if (p->ctx) cudaSetDevice(p->ctx->device);
    cudaStream_t s = p->ctx ? p->ctx->stream : nullptr;
    if (p->d_nprod) cudaFreeAsync(p->d_nprod, s);
    if (p->d_cnt) cudaFreeAsync(p->d_cnt, s);
    if (p->d_cptr) cudaFreeAsync(p->d_cptr, s);
    if (p->d_lists) cudaFreeAsync(p->d_lists, s);
    if (p->d_counters) cudaFreeAsync(p->d_counters, s);
    delete p;
    return SPRS_B200_OK;
}

}  // extern "C"
