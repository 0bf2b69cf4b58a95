// ldl.cu -- sparse LDL^T factorization L D L^T = P A P^T and its solve, for sm_90a.
//
// Replaces the sprs-ldl crate's LdlSymbolic / LdlNumeric (ldl_symbolic, ldl_numeric, ldl_lsolve,
// ldl_ltsolve, sprs-ldl/src/lib.rs) and sprs::is_symmetric (sprs/src/sparse/symmetric.rs).  The
// result is bit-identical to the reference: L's colptr, indices and values, D, x of `solve` and
// the first singular index.
//
// The up-looking algorithm.  Row k of P A P^T is the stored outer vector perm[k] of the matrix,
// its indices j mapped to pinv[j] in stored order.  Row k of L solves L[0:k,0:k] y = that row:
//   * y starts at +0.0 and each input entry with pinv[j] <= k does y_j = y_j + v; D_k = y_k;
//   * the pattern of row k: every input entry with pinv[j] < k contributes its elimination-tree
//     path from pinv[j] upward, stopping before the first node already listed; each path is
//     listed bottom-up and the paths in REVERSE stored-entry order;
//   * for each pattern node i in that order: y_j = y_j - L_ji * y_i over the entries of column i
//     written so far (rows j < k, ascending), then l_ki = y_i / D_i, D_k = D_k - l_ki * y_i, and
//     l_ki is appended to column i.
// Each multiply, subtraction and division is rounded on its own (--fmad=false).
//
// Design (DESIGN.md 4.9).
//   * SYMBOLIC, on the host, once per pattern: one serial walk over the rows gives the
//     elimination tree, every row's pattern in the order above and the column counts (the walk
//     is sequential by definition; a device mirror's indptr and indices are downloaded once for
//     it).  From the patterns: L's colptr and row indices (CSC, as the reference stores L), the
//     CSR of L's pattern (columns ascending per row), and for every pattern entry (k, i) its CSR
//     position and its CSC slot.  Entries [colptr[i], slot) of column i are then exactly the
//     rows j < k that row k reads.  |L| >= 2^32 is refused.
//   * NUMERIC (factor, update), one launch: one warp per row, rows claimed by a ticket counter
//     in ascending order.  Row k depends only on the rows of its pattern (all < k), so the
//     lowest unfinished ticket can always proceed, with no assumption on resident CTAs; the
//     warp waits on its pattern rows' ready flags with the progress-bounded waits of the
//     triangular solve (common.cuh, DESIGN.md 4.8).  y lives in the CSR value slots of row k:
//     a column-i entry j finds its slot by binary search in row k's sorted columns, so lanes
//     update distinct slots in parallel, and each slot is overwritten by l_ki once y_i is read.
//     No n-sized scratch per warp and no limit on the width of a row.  The chain of D_k and the
//     order of the pattern steps are serial, with __syncwarp between consecutive steps.  A row
//     ends with D_k, the CSC store of every l_ki (done per step) and a release store of its
//     flag.  The first k with D_k == 0.0 (-0.0 counts, NaN does not) is kept by atomicMin;
//     later rows may hold inf or NaN and are never exposed.  Each launch uses a new epoch.
//   * SOLVE: x = b[perm], the unit-diagonal lower solve on the CSR of L (the reference's column
//     sweep subtracts from x_j in ascending column order: the row sweep's order), x_i /= D_i,
//     the unit-diagonal upper solve on the CSC of L read as the CSR of L^T (column i in stored
//     order), out = x[pinv].  The two solves are the kernel of trisolve.cu.

#include "common.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <vector>

struct sprs_b200_ldl {
    sprs_b200_ctx* ctx = nullptr;
    const sprs_b200_ldl* sym = nullptr;  // numeric handles: the symbolic one (borrowed)
    uint64_t n = 0, nnz_l = 0;
    // symbolic: the input's pattern (copies), the permutation, L's structure
    uint64_t a_nnz = 0, a_outer = 0;
    int a_ipb = 4;
    Owned<void> d_a_ip;
    Owned<uint32_t> d_a_idx;
    Owned<uint32_t> d_perm, d_pinv;
    Owned<uint32_t> d_colptr, d_lidx;       // CSC of L
    Owned<uint32_t> d_rowptr, d_cidx;       // CSR of L's pattern
    Owned<uint32_t> d_pat_pos, d_pat_slot;  // per pattern entry, pattern order
    // numeric
    Owned<double> d_lcsr, d_lcsc, d_diag, d_tmp;
    Owned<uint32_t> d_flags;
    Owned<unsigned long long> d_words;     // [0] ticket counter, [1] first singular row
    Owned<unsigned long long> d_progress;  // per warp of the launch
    uint64_t n_progress = 0;
    Owned<unsigned long long> h_err;       // pinned: a wait bound was exceeded
    cudaEvent_t ev_last = nullptr;
    uint32_t epoch = 0;
    int state = 0;  // numeric: 0 factor valid, 1 singular (sing_index), 2 no valid factor
    uint64_t sing_index = 0;
    sprs_b200_csmat l_csr, lt_csr;  // borrowed views of L and L^T for the solves
    sprs_b200_trisolve *plan_l = nullptr, *plan_lt = nullptr;
};

namespace {

constexpr int LDL_THREADS = 256;
constexpr unsigned LDL_CTAS_PER_SM = 8;
constexpr uint32_t NO_PARENT = 0xffffffffu;

__device__ __forceinline__ uint64_t ip_at(const void* ip, int bytes, uint64_t i) {
    return bytes == 4 ? ((const uint32_t*)ip)[i] : ((const uint64_t*)ip)[i];
}

// position of column j in the sorted columns [lo, hi) (present by construction)
__device__ __forceinline__ uint32_t find_col(const uint32_t* __restrict__ cidx, uint32_t lo,
                                             uint32_t hi, uint32_t j) {
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (__ldg(cidx + mid) < j)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

template <typename P>
struct LdlArgs {
    const P* ip;             // the input matrix (outer vectors)
    const uint32_t* idx;
    const double* val;
    const uint32_t* perm;
    const uint32_t* pinv;
    const uint32_t* rowptr;  // CSR of L's pattern
    const uint32_t* cidx;
    const uint32_t* pat_pos;
    const uint32_t* pat_slot;
    const uint32_t* colptr;  // CSC of L
    const uint32_t* lidx;
    double* y;               // CSR values: y during row k, then L_k*
    double* lcsc;            // CSC values
    double* diag;
    uint32_t* flags;
    unsigned long long* ticket;
    unsigned long long* key;
    unsigned long long* err;
    unsigned long long* progress;
    uint64_t n_progress;
    uint64_t n;
    uint32_t epoch;
};

template <typename P>
__global__ void __launch_bounds__(LDL_THREADS) ldl_numeric_kernel(LdlArgs<P> a) {
    const unsigned lane = threadIdx.x & 31;
    unsigned long long* mine = a.progress + blockIdx.x * (LDL_THREADS / 32) + threadIdx.x / 32;
    unsigned long long done = 0;  // this warp's rows and heartbeats
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(a.ticket, 1ull);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= a.n) return;
        const uint32_t k = (uint32_t)t;
        const uint32_t rs = __ldg(a.rowptr + k), re = __ldg(a.rowptr + k + 1);
        // y = +0.0 on row k's pattern, then y_j = y_j + v for the input entries
        for (uint32_t p = rs + lane; p < re; p += 32) __stcg(a.y + p, 0.0);
        __syncwarp();
        const uint32_t o = __ldg(a.perm + k);
        const uint64_t s = a.ip[o], e = a.ip[o + 1];
        double yk = 0.0;
        bool has_k = false;
        for (uint64_t p = s + lane; p < e; p += 32) {
            const uint32_t j = __ldg(a.pinv + __ldg(a.idx + p));
            const double v = __dadd_rn(0.0, __ldg(a.val + p));
            if (j < k) {
                __stcg(a.y + find_col(a.cidx, rs, re, j), v);
            } else if (j == k) {
                yk = v;
                has_k = true;
            }
        }
        const unsigned kb = __ballot_sync(0xffffffffu, has_k);
        double dk = kb ? __shfl_sync(0xffffffffu, yk, __ffs(kb) - 1) : 0.0;
        // every row of the pattern, and so every row of the column prefixes read, is done
        bool ok = true;
        for (uint32_t p = rs + lane; p < re; p += 32)
            ok = ok && wait_ready(a.flags + __ldg(a.cidx + p), a.epoch, a.progress, a.n_progress);
        if (__any_sync(0xffffffffu, !ok)) {
            if (lane == 0) *(volatile unsigned long long*)a.err = 1ull;
            return;
        }
        __syncwarp();
        for (uint32_t base = rs; base < re; base += 32) {
            uint32_t my_pos = 0, my_slot = 0, my_col = 0;
            if (base + lane < re) {
                my_pos = __ldg(a.pat_pos + base + lane);
                my_slot = __ldg(a.pat_slot + base + lane);
                my_col = __ldg(a.cidx + my_pos);
            }
            const int cnt = re - base < 32 ? (int)(re - base) : 32;
            for (int st = 0; st < cnt; ++st) {
                const uint32_t pos = __shfl_sync(0xffffffffu, my_pos, st);
                const uint32_t slot = __shfl_sync(0xffffffffu, my_slot, st);
                const uint32_t i = __shfl_sync(0xffffffffu, my_col, st);
                // lane 0 overwrites y_i with l_ki below: every lane takes y_i from lane 0's
                // read, which precedes that store
                const double yi = __shfl_sync(0xffffffffu, __ldcg(a.y + pos), 0);
                for (uint32_t q = __ldg(a.colptr + i) + lane; q < slot; q += 32) {
                    const uint32_t pj = find_col(a.cidx, rs, re, __ldg(a.lidx + q));
                    __stcg(a.y + pj, __dsub_rn(__ldcg(a.y + pj), __dmul_rn(__ldcg(a.lcsc + q), yi)));
                }
                if (lane == 0) {
                    const double lki = __ddiv_rn(yi, __ldcg(a.diag + i));
                    dk = __dsub_rn(dk, __dmul_rn(lki, yi));
                    __stcg(a.y + pos, lki);
                    __stcg(a.lcsc + slot, lki);
                }
                __syncwarp();
            }
            if (lane == 0 && base + 32 < re) __stcg(mine, ++done);
        }
        if (lane == 0) {
            __stcg(a.diag + k, dk);
            if (dk == 0.0) atomicMin(a.key, (unsigned long long)k);  // -0.0 == 0.0; NaN != 0.0
            st_release_u32(a.flags + k, a.epoch);
            __stcg(mine, ++done);
        }
    }
}

// is_symmetric: every entry has a transposed partner with an equal value (== : NaN fails)
template <typename P>
__global__ void __launch_bounds__(LDL_THREADS)
symmetric_kernel(const P* __restrict__ ip, const uint32_t* __restrict__ idx,
                 const double* __restrict__ val, uint64_t n, unsigned* __restrict__ bad) {
    const uint64_t o = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) / 32;
    const unsigned lane = threadIdx.x & 31;
    if (o >= n) return;
    for (uint64_t p = ip[o] + lane; p < ip[o + 1]; p += 32) {
        const uint32_t i = idx[p];
        uint64_t lo = ip[i], hi = ip[i + 1];
        const uint64_t end = hi;
        while (lo < hi) {
            const uint64_t mid = lo + (hi - lo) / 2;
            if (idx[mid] < o)
                lo = mid + 1;
            else
                hi = mid;
        }
        if (!(lo < end && idx[lo] == o && val[lo] == val[p])) atomicOr(bad, 1u);
    }
}

// *bad = 1 where pattern a (the matrix given) differs from b (the symbolic factorization's);
// device mirrors are zero-based
__global__ void pattern_diff_kernel(const void* __restrict__ ip_a, int ipb_a,
                                    const uint32_t* __restrict__ idx_a,
                                    const void* __restrict__ ip_b, int ipb_b,
                                    const uint32_t* __restrict__ idx_b, uint64_t outer,
                                    uint64_t nnz, unsigned* __restrict__ bad) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= outer; i += stride)
        if (ip_at(ip_a, ipb_a, i) != ip_at(ip_b, ipb_b, i)) atomicOr(bad, 1u);
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz; i += stride)
        if (idx_a[i] != idx_b[i]) atomicOr(bad, 1u);
}

// x[i] = b[p[i]]: `&perm * b` of the reference (permutation.rs)
__global__ void permute_kernel(const double* __restrict__ b, const uint32_t* __restrict__ p,
                               double* __restrict__ x, uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) x[i] = b[p[i]];
}

// linalg::diag_solve: x_i = x_i / d_i
__global__ void diag_solve_kernel(const double* __restrict__ d, double* __restrict__ x,
                                  uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) x[i] = __ddiv_rn(x[i], d[i]);
}

unsigned blocks_for(uint64_t n, unsigned threads) {
    return (unsigned)std::max<uint64_t>(1, (n + threads - 1) / threads);
}

template <typename T>
int upload(sprs_b200_ctx* ctx, const std::vector<T>& h, Owned<T>* d) {
    SPRS_TRY(d->alloc(ctx, h.size() * sizeof(T) + 16, "ldl symbolic"));
    if (!h.empty())
        SPRS_CUDA(ctx, cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    return SPRS_B200_OK;
}

int is_symmetric_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, bool* sym) {
    *sym = false;
    if (m->rows != m->cols) return SPRS_B200_OK;
    cudaStream_t s = ctx->stream;
    void* d_bad = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 3, sizeof(unsigned), &d_bad));
    SPRS_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(unsigned), s));
    if (m->outer) {
        const unsigned g = blocks_for(m->outer * 32, LDL_THREADS);
        if (m->indptr_bytes == 4)
            symmetric_kernel<uint32_t><<<g, LDL_THREADS, 0, s>>>(
                (const uint32_t*)m->d_indptr, m->d_indices, m->d_data, m->outer, (unsigned*)d_bad);
        else
            symmetric_kernel<uint64_t><<<g, LDL_THREADS, 0, s>>>(
                (const uint64_t*)m->d_indptr, m->d_indices, m->d_data, m->outer, (unsigned*)d_bad);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaGetLastError());
    }
    unsigned bad = 0;
    SPRS_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    *sym = bad == 0;
    return SPRS_B200_OK;
}

// The host walk: elimination tree, row patterns in the reference's order, L's structure.
struct Structure {
    std::vector<uint32_t> colptr, lidx, rowptr, cidx, pat_pos, pat_slot;
};

template <typename P>
int analyse(sprs_b200_ctx* ctx, const std::vector<P>& ip, const std::vector<uint32_t>& idx,
            const std::vector<uint32_t>& perm, const std::vector<uint32_t>& pinv, Structure* out) {
    const uint64_t n = perm.size();
    std::vector<uint32_t> parent(n, NO_PARENT), flag(n), count(n, 0), pat;
    std::vector<uint64_t> paths;  // (start, end) of each path of the current row
    std::vector<uint32_t> tmp;
    out->rowptr.assign(n + 1, 0);
    for (uint64_t k = 0; k < n; ++k) {
        flag[k] = (uint32_t)k;
        const uint64_t row_start = pat.size();
        paths.clear();
        const uint32_t o = perm[k];
        for (P p = ip[o]; p < ip[o + 1]; ++p) {
            uint32_t i = pinv[idx[p]];
            if (i >= k) continue;
            const uint64_t ps = pat.size();
            while (flag[i] != k) {
                if (parent[i] == NO_PARENT) parent[i] = (uint32_t)k;
                count[i] += 1;
                flag[i] = (uint32_t)k;
                pat.push_back(i);
                i = parent[i];
            }
            if (pat.size() > ps) {
                paths.push_back(ps);
                paths.push_back(pat.size());
            }
        }
        if (pat.size() >= 0xffffffffull)
            SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE,
                      "ldl: L has 2^32 or more non-zeros (u32 index arrays)");
        if (paths.size() > 2) {  // the paths in reverse stored-entry order, each bottom-up
            tmp.assign(pat.begin() + row_start, pat.end());
            uint64_t w = row_start;
            for (uint64_t q = paths.size(); q >= 2; q -= 2)
                for (uint64_t x = paths[q - 2]; x < paths[q - 1]; ++x) pat[w++] = tmp[x - row_start];
        }
        out->rowptr[k + 1] = (uint32_t)pat.size();
    }
    const uint64_t nnz = pat.size();
    // CSC of L: row k appended to column i for each pattern entry, rows ascending
    out->colptr.assign(n + 1, 0);
    for (uint64_t i = 0; i < n; ++i) out->colptr[i + 1] = out->colptr[i] + count[i];
    std::vector<uint32_t> fill(out->colptr.begin(), out->colptr.end() - (n ? 1 : 0));
    out->lidx.resize(nnz);
    out->pat_slot.resize(nnz);
    for (uint64_t k = 0; k < n; ++k)
        for (uint32_t p = out->rowptr[k]; p < out->rowptr[k + 1]; ++p) {
            const uint32_t slot = fill[pat[p]]++;
            out->lidx[slot] = (uint32_t)k;
            out->pat_slot[p] = slot;
        }
    // CSR of L's pattern (columns ascending per row) and the CSR position of every CSC slot
    std::vector<uint32_t> pos_of_slot(nnz), next(out->rowptr.begin(), out->rowptr.end() - (n ? 1 : 0));
    out->cidx.resize(nnz);
    for (uint64_t i = 0; i < n; ++i)
        for (uint32_t q = out->colptr[i]; q < out->colptr[i + 1]; ++q) {
            const uint32_t at = next[out->lidx[q]]++;
            out->cidx[at] = (uint32_t)i;
            pos_of_slot[q] = at;
        }
    out->pat_pos.resize(nnz);
    for (uint64_t p = 0; p < nnz; ++p) out->pat_pos[p] = pos_of_slot[out->pat_slot[p]];
    return SPRS_B200_OK;
}

void free_ldl(sprs_b200_ldl* h) {
    if (h->ctx) cudaSetDevice(h->ctx->device);
    if (h->plan_l) sprs_b200_trisolve_free(h->plan_l);
    if (h->plan_lt) sprs_b200_trisolve_free(h->plan_lt);
    if (h->ev_last) cudaEventDestroy(h->ev_last);
    delete h;
}
using LdlPtr = std::unique_ptr<sprs_b200_ldl, FreeWith<free_ldl>>;

template <typename P>
int build_symbolic(sprs_b200_ldl* h, const sprs_b200_csmat* m, const std::vector<uint32_t>& perm) {
    sprs_b200_ctx* ctx = h->ctx;
    const uint64_t n = h->n;
    std::vector<P> ip(m->outer + 1);
    std::vector<uint32_t> idx(m->nnz);
    SPRS_CUDA(ctx, cudaMemcpy(ip.data(), m->d_indptr, ip.size() * sizeof(P), cudaMemcpyDeviceToHost));
    if (m->nnz)
        SPRS_CUDA(ctx, cudaMemcpy(idx.data(), m->d_indices, m->nnz * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost));
    std::vector<uint32_t> pinv(n);
    for (uint64_t i = 0; i < n; ++i) pinv[perm[i]] = (uint32_t)i;
    Structure st;
    SPRS_TRY(analyse<P>(ctx, ip, idx, perm, pinv, &st));
    h->nnz_l = st.lidx.size();
    SPRS_TRY(upload(ctx, perm, &h->d_perm));
    SPRS_TRY(upload(ctx, pinv, &h->d_pinv));
    SPRS_TRY(upload(ctx, st.colptr, &h->d_colptr));
    SPRS_TRY(upload(ctx, st.lidx, &h->d_lidx));
    SPRS_TRY(upload(ctx, st.rowptr, &h->d_rowptr));
    SPRS_TRY(upload(ctx, st.cidx, &h->d_cidx));
    SPRS_TRY(upload(ctx, st.pat_pos, &h->d_pat_pos));
    SPRS_TRY(upload(ctx, st.pat_slot, &h->d_pat_slot));
    // the pattern `update` is checked against
    h->a_nnz = m->nnz;
    h->a_outer = m->outer;
    h->a_ipb = m->indptr_bytes;
    SPRS_TRY(h->d_a_ip.alloc(ctx, ip.size() * sizeof(P), "ldl symbolic"));
    SPRS_TRY(h->d_a_idx.alloc(ctx, m->nnz * sizeof(uint32_t) + 16, "ldl symbolic"));
    SPRS_CUDA(ctx, cudaMemcpy(h->d_a_ip, ip.data(), ip.size() * sizeof(P), cudaMemcpyHostToDevice));
    if (m->nnz)
        SPRS_CUDA(ctx, cudaMemcpy(h->d_a_idx, idx.data(), m->nnz * sizeof(uint32_t),
                                  cudaMemcpyHostToDevice));
    return SPRS_B200_OK;
}

int alloc_numeric(sprs_b200_ldl* h) {
    sprs_b200_ctx* ctx = h->ctx;
    const sprs_b200_ldl* sy = h->sym;
    const uint64_t n = h->n, nnz = h->nnz_l;
    SPRS_TRY(h->d_lcsr.alloc(ctx, nnz * sizeof(double) + 16, "ldl factor"));
    SPRS_TRY(h->d_lcsc.alloc(ctx, nnz * sizeof(double) + 16, "ldl factor"));
    SPRS_TRY(h->d_diag.alloc(ctx, n * sizeof(double) + 16, "ldl factor"));
    SPRS_TRY(h->d_tmp.alloc(ctx, n * sizeof(double) + 16, "ldl factor"));
    SPRS_TRY(h->d_flags.alloc(ctx, n * sizeof(uint32_t) + 16, "ldl factor"));
    SPRS_CUDA(ctx, cudaMemset(h->d_flags, 0, n * sizeof(uint32_t) + 16));
    SPRS_TRY(h->d_words.alloc(ctx, 2 * sizeof(unsigned long long), "ldl factor"));
    h->n_progress = (uint64_t)ctx->sm_count * LDL_CTAS_PER_SM * (LDL_THREADS / 32);
    SPRS_TRY(h->d_progress.alloc(ctx, h->n_progress * sizeof(unsigned long long), "ldl factor"));
    SPRS_TRY(h->h_err.alloc_pinned(ctx, sizeof(unsigned long long), "ldl factor"));
    *h->h_err = 0;
    SPRS_CUDA(ctx, cudaEventCreateWithFlags(&h->ev_last, cudaEventDisableTiming));
    // L (CSR, unit lower) and L^T (the CSC arrays read as CSR, unit upper) for the solves
    h->l_csr = csmat_init(ctx, SPRS_B200_CSR, n, n, nnz, 4, Arrays::borrowed);
    h->lt_csr = csmat_init(ctx, SPRS_B200_CSR, n, n, nnz, 4, Arrays::borrowed);
    h->l_csr.d_indptr = sy->d_rowptr;
    h->l_csr.d_indices = sy->d_cidx;
    h->l_csr.d_data = h->d_lcsr;
    h->lt_csr.d_indptr = sy->d_colptr;
    h->lt_csr.d_indices = sy->d_lidx;
    h->lt_csr.d_data = h->d_lcsc;
    SPRS_TRY(trisolve_unit_plan(ctx, &h->l_csr, SPRS_B200_TRI_LOWER, &h->plan_l));
    SPRS_TRY(trisolve_unit_plan(ctx, &h->lt_csr, SPRS_B200_TRI_UPPER, &h->plan_lt));
    return SPRS_B200_OK;
}

template <typename P>
void launch_numeric(sprs_b200_ldl* h, const sprs_b200_csmat* m, unsigned g, cudaStream_t s) {
    const sprs_b200_ldl* sy = h->sym;
    LdlArgs<P> a;
    a.ip = (const P*)m->d_indptr;
    a.idx = m->d_indices;
    a.val = m->d_data;
    a.perm = sy->d_perm;
    a.pinv = sy->d_pinv;
    a.rowptr = sy->d_rowptr;
    a.cidx = sy->d_cidx;
    a.pat_pos = sy->d_pat_pos;
    a.pat_slot = sy->d_pat_slot;
    a.colptr = sy->d_colptr;
    a.lidx = sy->d_lidx;
    a.y = h->d_lcsr;
    a.lcsc = h->d_lcsc;
    a.diag = h->d_diag;
    a.flags = h->d_flags;
    a.ticket = h->d_words;
    a.key = h->d_words + 1;
    a.err = h->h_err;
    a.progress = h->d_progress;
    a.n_progress = (uint64_t)g * (LDL_THREADS / 32);
    a.n = h->n;
    a.epoch = h->epoch;
    ldl_numeric_kernel<P><<<g, LDL_THREADS, 0, s>>>(a);
}

// ldl_numeric on the device; blocking.  ERR_STRUCTURE (nothing launched but the comparison)
// when the matrix's pattern is not the symbolic factorization's.
int numeric(sprs_b200_ldl* h, const sprs_b200_csmat* m) {
    sprs_b200_ctx* ctx = h->ctx;
    const sprs_b200_ldl* sy = h->sym;
    cudaStream_t s = ctx->stream;
    if (m->rows != h->n || m->cols != h->n)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    bool same = m->nnz == sy->a_nnz && m->outer == sy->a_outer;
    if (same) {
        void* d_bad = nullptr;
        SPRS_TRY(ctx_scratch(ctx, 3, sizeof(unsigned), &d_bad));
        SPRS_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(unsigned), s));
        pattern_diff_kernel<<<std::min(blocks_for(m->nnz + m->outer + 1, LDL_THREADS), 4096u),
                              LDL_THREADS, 0, s>>>(m->d_indptr, m->indptr_bytes, m->d_indices,
                                                   sy->d_a_ip, sy->a_ipb, sy->d_a_idx, m->outer,
                                                   m->nnz, (unsigned*)d_bad);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaGetLastError());
        unsigned bad = 0;
        SPRS_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, s));
        SPRS_CUDA(ctx, cudaStreamSynchronize(s));
        same = bad == 0;
    }
    if (!same)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STRUCTURE,
                  "ldl update: the matrix's pattern differs from the symbolic factorization's");
    // the solves of the previous factor are done before its values are overwritten
    SPRS_CUDA(ctx, cudaStreamWaitEvent(s, h->ev_last, 0));
    h->state = 2;
    if (h->n) {
        if (++h->epoch == 0) {
            SPRS_CUDA(ctx, cudaMemsetAsync(h->d_flags, 0, h->n * sizeof(uint32_t), s));
            h->epoch = 1;
        }
        const unsigned long long init[2] = {0ull, ~0ull};
        SPRS_CUDA(ctx, cudaMemcpyAsync(h->d_words, init, sizeof(init), cudaMemcpyHostToDevice, s));
        const uint64_t warps = LDL_THREADS / 32;
        const unsigned g = (unsigned)std::min<uint64_t>((h->n + warps - 1) / warps,
                                                        (uint64_t)ctx->sm_count * LDL_CTAS_PER_SM);
        SPRS_CUDA(ctx, cudaMemsetAsync(h->d_progress, 0, g * warps * sizeof(unsigned long long), s));
        if (m->indptr_bytes == 4)
            launch_numeric<uint32_t>(h, m, g, s);
        else
            launch_numeric<uint64_t>(h, m, g, s);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaGetLastError());
        unsigned long long key = 0;
        SPRS_CUDA(ctx, cudaMemcpyAsync(&key, h->d_words + 1, sizeof(key), cudaMemcpyDeviceToHost, s));
        SPRS_CUDA(ctx, cudaStreamSynchronize(s));
        if (*(volatile unsigned long long*)h->h_err) {
            *(volatile unsigned long long*)h->h_err = 0;
            SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA,
                      "ldl: no row of the factorization progressed for the wait bound");
        }
        if (key != ~0ull) {
            h->state = 1;
            h->sing_index = key;
            SPRS_FAIL(ctx, SPRS_B200_ERR_SINGULAR,
                      "Singular matrix at index %llu (diagonal element is a numeric 0)", key);
        }
    }
    h->state = 0;
    return SPRS_B200_OK;
}

int require_factor(const sprs_b200_ldl* h) {
    if (!h->sym) SPRS_FAIL(h->ctx, SPRS_B200_ERR_ARGUMENT, "ldl: a symbolic handle has no factor");
    if (h->state == 1)
        SPRS_FAIL(h->ctx, SPRS_B200_ERR_SINGULAR,
                  "Singular matrix at index %llu (diagonal element is a numeric 0)",
                  (unsigned long long)h->sing_index);
    if (h->state != 0)
        SPRS_FAIL(h->ctx, SPRS_B200_ERR_ARGUMENT, "ldl: the last update failed; no valid factor");
    return SPRS_B200_OK;
}

int enqueue_solve(sprs_b200_ldl* h, const double* d_b, double* d_x, cudaStream_t s) {
    sprs_b200_ctx* ctx = h->ctx;
    const uint64_t n = h->n;
    if (!n) return SPRS_B200_OK;
    const unsigned g = blocks_for(n, LDL_THREADS);
    permute_kernel<<<g, LDL_THREADS, 0, s>>>(d_b, h->sym->d_perm, h->d_tmp, n);
    SPRS_TRY(trisolve_enqueue(h->plan_l, h->d_tmp, s));
    diag_solve_kernel<<<g, LDL_THREADS, 0, s>>>(h->d_diag, h->d_tmp, n);
    SPRS_TRY(trisolve_enqueue(h->plan_lt, h->d_tmp, s));
    permute_kernel<<<g, LDL_THREADS, 0, s>>>(h->d_tmp, h->sym->d_pinv, d_x, n);
    ctx->launches += 3;
    SPRS_CUDA(ctx, cudaGetLastError());
    SPRS_CUDA(ctx, cudaEventRecord(h->ev_last, s));
    return SPRS_B200_OK;
}

}  // namespace

extern "C" {

int sprs_b200_is_symmetric(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, int* out) {
    if (!ctx || !mat || !out) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    bool sym = false;
    SPRS_TRY(is_symmetric_dev(ctx, mat, &sym));
    *out = sym ? 1 : 0;
    return SPRS_B200_OK;
}

int sprs_b200_diag_solve(sprs_b200_ctx* ctx, const double* diag, double* x, uint64_t len) {
    if (!ctx || (len && (!diag || !x))) return SPRS_B200_ERR_ARGUMENT;
    if (!len) return SPRS_B200_OK;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    void *d_d = nullptr, *d_x = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 0, len * sizeof(double), &d_d));
    SPRS_TRY(ctx_scratch(ctx, 1, len * sizeof(double), &d_x));
    SPRS_CUDA(ctx, cudaMemcpyAsync(d_d, diag, len * sizeof(double), cudaMemcpyHostToDevice, s));
    SPRS_CUDA(ctx, cudaMemcpyAsync(d_x, x, len * sizeof(double), cudaMemcpyHostToDevice, s));
    diag_solve_kernel<<<blocks_for(len, LDL_THREADS), LDL_THREADS, 0, s>>>((const double*)d_d,
                                                                          (double*)d_x, len);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    SPRS_CUDA(ctx, cudaMemcpyAsync(x, d_x, len * sizeof(double), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    return SPRS_B200_OK;
}

int sprs_b200_ldl_symbolic(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const uint32_t* perm,
                           int check_symmetry, sprs_b200_ldl** out) {
    if (!ctx || !mat || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if (mat->rows != mat->cols) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "matrix should be square");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    if (check_symmetry) {
        bool sym = false;
        SPRS_TRY(is_symmetric_dev(ctx, mat, &sym));
        if (!sym) SPRS_FAIL(ctx, SPRS_B200_ERR_NOT_SYMMETRIC, "Matrix is not symmetric");
    }
    const uint64_t n = mat->rows;
    std::vector<uint32_t> p(n);
    if (perm) {
        std::vector<char> seen(n, 0);
        for (uint64_t i = 0; i < n; ++i) {
            if (perm[i] >= n || seen[perm[i]])
                SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "assertion failed: perm_is_valid(&perm)");
            seen[perm[i]] = 1;
            p[i] = perm[i];
        }
    } else {
        for (uint64_t i = 0; i < n; ++i) p[i] = (uint32_t)i;
    }
    LdlPtr h(new sprs_b200_ldl());
    h->ctx = ctx;
    h->n = n;
    SPRS_TRY(mat->indptr_bytes == 4 ? build_symbolic<uint32_t>(h.get(), mat, p)
                                    : build_symbolic<uint64_t>(h.get(), mat, p));
    *out = h.release();
    return SPRS_B200_OK;
}

uint64_t sprs_b200_ldl_nnz(const sprs_b200_ldl* ldl) {
    return ldl ? ldl->nnz_l : 0;
}

int sprs_b200_ldl_factor(const sprs_b200_ldl* sym, const sprs_b200_csmat* mat, sprs_b200_ldl** out) {
    if (!sym || !mat || !out || sym->sym) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    sprs_b200_ctx* ctx = sym->ctx;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    LdlPtr h(new sprs_b200_ldl());
    h->ctx = ctx;
    h->sym = sym;
    h->n = sym->n;
    h->nnz_l = sym->nnz_l;
    h->state = 2;
    SPRS_TRY(alloc_numeric(h.get()));
    const int st = numeric(h.get(), mat);
    if (st != SPRS_B200_OK && st != SPRS_B200_ERR_SINGULAR) return st;
    *out = h.release();
    return st;
}

int sprs_b200_ldl_update(sprs_b200_ldl* num, const sprs_b200_csmat* mat) {
    if (!num || !mat || !num->sym) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(num->ctx, cudaSetDevice(num->ctx->device));
    return numeric(num, mat);
}

int sprs_b200_ldl_singular(const sprs_b200_ldl* num, uint64_t* index) {
    if (!num || num->state != 1) return 0;
    if (index) *index = num->sing_index;
    return 1;
}

int sprs_b200_ldl_solve(sprs_b200_ldl* num, const double* b, double* x, uint64_t len) {
    if (!num) return SPRS_B200_ERR_ARGUMENT;
    SPRS_TRY(require_factor(num));
    sprs_b200_ctx* ctx = num->ctx;
    if (len != num->n) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (len && (!b || !x)) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    void* d_v = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 1, len * sizeof(double), &d_v));
    if (len) SPRS_CUDA(ctx, cudaMemcpyAsync(d_v, b, len * sizeof(double), cudaMemcpyHostToDevice, s));
    SPRS_TRY(enqueue_solve(num, (const double*)d_v, (double*)d_v, s));
    if (len) SPRS_CUDA(ctx, cudaMemcpyAsync(x, d_v, len * sizeof(double), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    SPRS_TRY(trisolve_check_breach(num->plan_l));
    return trisolve_check_breach(num->plan_lt);
}

int sprs_b200_ldl_solve_dev(sprs_b200_ldl* num, const double* d_b, double* d_x, void* stream) {
    if (!num) return SPRS_B200_ERR_ARGUMENT;
    SPRS_TRY(require_factor(num));
    if (num->n && (!d_b || !d_x)) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(num->ctx, cudaSetDevice(num->ctx->device));
    return enqueue_solve(num, d_b, d_x, pick_stream(num->ctx, stream));
}

int sprs_b200_ldl_get_l(const sprs_b200_ldl* num, uint32_t* colptr, uint32_t* indices,
                        double* data) {
    if (!num) return SPRS_B200_ERR_ARGUMENT;
    SPRS_TRY(require_factor(num));
    sprs_b200_ctx* ctx = num->ctx;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (colptr)
        SPRS_CUDA(ctx, cudaMemcpy(colptr, num->sym->d_colptr, (num->n + 1) * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost));
    if (indices && num->nnz_l)
        SPRS_CUDA(ctx, cudaMemcpy(indices, num->sym->d_lidx, num->nnz_l * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost));
    if (data && num->nnz_l)
        SPRS_CUDA(ctx, cudaMemcpy(data, num->d_lcsc, num->nnz_l * sizeof(double),
                                  cudaMemcpyDeviceToHost));
    return SPRS_B200_OK;
}

int sprs_b200_ldl_get_d(const sprs_b200_ldl* num, double* d, uint64_t len) {
    if (!num) return SPRS_B200_ERR_ARGUMENT;
    SPRS_TRY(require_factor(num));
    sprs_b200_ctx* ctx = num->ctx;
    if (len != num->n) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (len) SPRS_CUDA(ctx, cudaMemcpy(d, num->d_diag, len * sizeof(double), cudaMemcpyDeviceToHost));
    return SPRS_B200_OK;
}

int sprs_b200_ldl_free(sprs_b200_ldl* ldl) {
    if (!ldl) return SPRS_B200_OK;
    cudaSetDevice(ldl->ctx->device);
    if (ldl->ev_last) {  // the last solve_dev, on whatever stream, may still use the factor
        cudaStreamWaitEvent(ldl->ctx->stream, ldl->ev_last, 0);
        cudaStreamSynchronize(ldl->ctx->stream);
    }
    free_ldl(ldl);
    return SPRS_B200_OK;
}

}  // extern "C"
