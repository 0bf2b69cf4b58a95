// trisolve.cu -- sparse triangular solves L x = b and U x = b with a dense right-hand side, for
// sm_90a.
//
// Replaces sprs::linalg::trisolve's lsolve_csr_dense_rhs, usolve_csr_dense_rhs,
// lsolve_csc_dense_rhs and usolve_csc_dense_rhs (sprs/src/sparse/linalg/trisolve.rs:30-262).
// Every row r is x = b_r; x = x - (a_rc * x_c) over its terms; x / diag, each multiply,
// subtraction and division rounded on its own (--fmad=false), the terms in the reference's
// order: ascending column, except usolve_csc, whose column sweep subtracts the terms of row r
// in DESCENDING column order.  A CSC matrix is solved on its CSR transpose (the same matrix in
// the other storage), so one kernel serves all four forms.  The result is bit-identical.
//
// Design (DESIGN.md 4.8).
//   * PLAN, once per matrix and triangle: the position of every row's diagonal (a binary search
//     per row) and the first singular row in processing order (diagonal missing or == 0, an
//     atomicMin over rows).  It reads the values: the mirror must not change while it lives.
//   * SOLVE: one warp per row.  Rows are claimed through a global ticket counter in processing
//     order (ascending rows for L, descending for U).  A row depends only on rows with smaller
//     tickets, and every claimed ticket is held by a warp that is running, so the lowest
//     unfinished ticket can always proceed: progress needs no assumption about how many CTAs
//     are resident (the GPU may be shared; the CPU emulator runs CTAs one after another).
//     Each group of 32 terms: lanes load (col, val), wait until row col's flag holds this
//     solve's epoch (acquire loads, __nanosleep backoff), load x_col through L2 (x is written
//     during the kernel: never the non-coherent path) and form the products in parallel; the
//     subtraction chain then runs serially in the reference's order through shuffles.  The row
//     ends with a store of x_r and a release store of its flag.  Flags are never cleared: each
//     solve uses a new epoch.
//   * SINGULAR at ticket k: the same launch solves the rows before k; CSC forms then leave in
//     rows from k on b_r minus the terms of the columns processed before k (no division, no
//     flag), as the reference's column sweep does when it returns early.
//   * Waits are bounded by PROGRESS, not by their own length: a legitimate wait can last almost
//     the whole solve (in an upper R-MAT solve the hub rows are claimed together and each waits
//     for the next, seconds in all).  Every warp counts its finished rows and every 256 groups
//     of a long row in a word of its own (a plain store, no shared atomic on the row path); a
//     wait that passes 2^34 clock64 cycles (~9 s at 1.98 GHz) takes the sum of those words and
//     gives up only if a further 2^34 cycles pass without the sum changing, i.e. when no warp
//     of the solve moved at all -- a bug, never a valid input.  A breach writes an error word
//     and the warp exits; the call then fails with ERR_CUDA.
//   * The subtraction chain of a row is serial by definition: a row of 10^6 terms is a 10^6
//     long dependent chain here as on the CPU.

#include "common.cuh"
#include "ptx.cuh"

#include <algorithm>

struct sprs_b200_trisolve {
    sprs_b200_ctx* ctx = nullptr;
    const sprs_b200_csmat* csr = nullptr;  // the rows solved: the mirror (CSR) or own_t (CSC)
    sprs_b200_csmat* own_t = nullptr;      // CSC mirrors: the device transpose
    int storage = SPRS_B200_CSR, tri = SPRS_B200_TRI_LOWER;
    uint64_t n = 0;
    uint32_t* d_diag = nullptr;            // per row: offset of the first entry with col >= r
    uint32_t* d_flags = nullptr;           // per row: epoch of the last solve that finished it
    unsigned long long* d_words = nullptr; // [0] ticket counter, [1] singular key (plan)
    unsigned long long* d_progress = nullptr;  // per warp of the solve: rows / heartbeats done
    uint64_t n_progress = 0;               // words in d_progress (warps of the largest grid)
    unsigned long long* h_err = nullptr;   // mapped pinned word: a wait bound was exceeded
    cudaEvent_t ev_last = nullptr;         // recorded behind the last enqueued solve
    uint32_t epoch = 0;
    uint64_t k_ticket = 0;                 // first singular ticket (n: none)
    uint64_t sing_index = 0;
    int sing_reason = 0;
    bool unit = false;                     // trisolve_unit_plan: no diagonal stored
};

namespace {

constexpr int TRI_THREADS = 256;
constexpr unsigned TRI_CTAS_PER_SM = 8;
constexpr uint64_t TRI_HEARTBEAT = 32 * 256;      // terms of a long row between progress ticks

template <typename P>
struct TriArgs {
    const P* ip;
    const uint32_t* idx;
    const double* val;
    const uint32_t* diag;
    uint32_t* flags;
    double* x;
    unsigned long long* ticket;
    unsigned long long* err;
    unsigned long long* progress;  // one word per warp of the launch
    uint64_t n_progress;
    uint64_t n;
    uint64_t k_ticket;  // first singular ticket (n: none)
    uint64_t n_work;    // tickets processed: k_ticket, or n for the CSC partial sums
    uint32_t epoch;
};

template <bool UPPER>
__device__ __forceinline__ uint64_t ticket_of(uint64_t r, uint64_t n) {
    return UPPER ? n - 1 - r : r;
}

template <typename P, bool UPPER>
__global__ void __launch_bounds__(TRI_THREADS)
trisolve_plan_kernel(const P* __restrict__ ip, const uint32_t* __restrict__ idx,
                     const double* __restrict__ val, uint64_t n, uint32_t* __restrict__ diag,
                     unsigned long long* __restrict__ key) {
    const uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint64_t s = ip[r], e = ip[r + 1];
    uint64_t lo = s, hi = e;  // first position with col >= r
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (idx[mid] < r)
            lo = mid + 1;
        else
            hi = mid;
    }
    diag[r] = (uint32_t)(lo - s);
    const bool present = lo < e && idx[lo] == r;
    if (!present || val[lo] == 0.0)  // -0.0 == 0.0; NaN != 0.0
        atomicMin(key, (unsigned long long)(ticket_of<UPPER>(r, n) << 1 | (present ? 1 : 0)));
}

// UPPER: rows in descending order, terms col > r.  REV: the terms of a row are subtracted in
// descending column order (usolve_csc).  UNIT: the rows hold only the triangle's terms and the
// diagonal is 1 (the L of an LDL^T factorization): no diagonal lookup, no division.
template <typename P, bool UPPER, bool REV, bool UNIT = false>
__global__ void __launch_bounds__(TRI_THREADS) trisolve_kernel(TriArgs<P> a) {
    const unsigned lane = threadIdx.x & 31;
    unsigned long long* mine = a.progress + blockIdx.x * (TRI_THREADS / 32) + threadIdx.x / 32;
    unsigned long long done = 0;  // this warp's rows and heartbeats
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(a.ticket, 1ull);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= a.n_work) return;
        const uint64_t r = UPPER ? a.n - 1 - t : t;
        const uint64_t s = a.ip[r], e = a.ip[r + 1];
        const uint64_t d = UNIT ? s : s + a.diag[r];  // first position with col >= r
        const bool solve = t < a.k_ticket;
        // the triangle's terms: [s, d) below the diagonal, (diagonal, e) above it
        uint64_t lo = s, hi = d;
        if (UNIT) {
            hi = e;
        } else if (UPPER) {
            lo = (d < e && a.idx[d] == r) ? d + 1 : d;
            hi = e;
        }
        const uint64_t len = hi - lo;
        double x = __ldcg(a.x + r);
        bool ok = true;
        for (uint64_t base = 0; base < len; base += 32) {
            const uint64_t j = base + lane;
            double p = 0.0;  // x - (+0.0) == x for every x: the identity of the chain
            if (j < len) {
                const uint64_t k = REV ? hi - 1 - j : lo + j;
                const uint32_t c = __ldg(a.idx + k);
                // rows from k_ticket on (CSC partial sums) take only the columns processed
                // before it; for the rows before it every term passes
                if (ticket_of<UPPER>(c, a.n) < a.k_ticket) {
                    ok = wait_ready(a.flags + c, a.epoch, a.progress, a.n_progress);
                    p = __dmul_rn(__ldg(a.val + k), __ldcg(a.x + c));
                }
            }
            if (__any_sync(0xffffffffu, !ok)) {
                if (lane == 0) *(volatile unsigned long long*)a.err = 1ull;
                return;
            }
            const int cnt = len - base < 32 ? (int)(len - base) : 32;
            for (int i = 0; i < cnt; ++i) x = __dsub_rn(x, __shfl_sync(0xffffffffu, p, i));
            if ((base + 32) % TRI_HEARTBEAT == 0 && lane == 0) __stcg(mine, ++done);
        }
        if (lane == 0) {
            if (solve && !UNIT) x = __ddiv_rn(x, __ldg(a.val + d));
            __stcg(a.x + r, x);
            if (solve) st_release_u32(a.flags + r, a.epoch);
            __stcg(mine, ++done);
        }
    }
}

template <typename P>
int launch_plan(sprs_b200_trisolve* p, cudaStream_t s) {
    const sprs_b200_csmat* m = p->csr;
    const unsigned g = (unsigned)((p->n + TRI_THREADS - 1) / TRI_THREADS);
    if (p->tri == SPRS_B200_TRI_UPPER)
        trisolve_plan_kernel<P, true><<<g, TRI_THREADS, 0, s>>>(
            (const P*)m->d_indptr, m->d_indices, m->d_data, p->n, p->d_diag, p->d_words + 1);
    else
        trisolve_plan_kernel<P, false><<<g, TRI_THREADS, 0, s>>>(
            (const P*)m->d_indptr, m->d_indices, m->d_data, p->n, p->d_diag, p->d_words + 1);
    p->ctx->launches += 1;
    SPRS_CUDA(p->ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

template <typename P>
int launch_solve(sprs_b200_trisolve* p, double* d_x, cudaStream_t s) {
    sprs_b200_ctx* ctx = p->ctx;
    const sprs_b200_csmat* m = p->csr;
    const bool csc = p->storage == SPRS_B200_CSC;
    TriArgs<P> a;
    a.ip = (const P*)m->d_indptr;
    a.idx = m->d_indices;
    a.val = m->d_data;
    a.diag = p->d_diag;
    a.flags = p->d_flags;
    a.x = d_x;
    a.ticket = p->d_words;
    a.err = p->h_err;
    a.progress = p->d_progress;
    a.n = p->n;
    a.k_ticket = p->k_ticket;
    a.n_work = csc ? p->n : p->k_ticket;
    a.epoch = p->epoch;
    if (a.n_work == 0) return SPRS_B200_OK;
    const uint64_t warps_per_cta = TRI_THREADS / 32;
    const unsigned g = (unsigned)std::min<uint64_t>((a.n_work + warps_per_cta - 1) / warps_per_cta,
                                                    (uint64_t)ctx->sm_count * TRI_CTAS_PER_SM);
    a.n_progress = (uint64_t)g * warps_per_cta;
    SPRS_CUDA(ctx, cudaMemsetAsync(p->d_words, 0, sizeof(unsigned long long), s));
    SPRS_CUDA(ctx, cudaMemsetAsync(p->d_progress, 0, a.n_progress * sizeof(unsigned long long), s));
    if (p->unit && p->tri == SPRS_B200_TRI_LOWER)
        trisolve_kernel<P, false, false, true><<<g, TRI_THREADS, 0, s>>>(a);
    else if (p->unit)
        trisolve_kernel<P, true, false, true><<<g, TRI_THREADS, 0, s>>>(a);
    else if (p->tri == SPRS_B200_TRI_LOWER)
        trisolve_kernel<P, false, false><<<g, TRI_THREADS, 0, s>>>(a);
    else if (csc)
        trisolve_kernel<P, true, true><<<g, TRI_THREADS, 0, s>>>(a);
    else
        trisolve_kernel<P, true, false><<<g, TRI_THREADS, 0, s>>>(a);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

// Enqueue one solve on `s` with a new epoch (flags are cleared only when the epoch wraps).
// A breach of the wait bound left by an earlier solve: reported once, then cleared (the next
// solve starts from a new epoch and a reset ticket counter, so the plan stays usable).
int take_breach(sprs_b200_trisolve* p, const char* when) {
    if (!*(volatile unsigned long long*)p->h_err) return SPRS_B200_OK;
    *(volatile unsigned long long*)p->h_err = 0;
    SPRS_FAIL(p->ctx, SPRS_B200_ERR_CUDA,
              "trisolve: no row of the solve progressed for the wait bound (%s); x is incomplete",
              when);
}

int enqueue_solve(sprs_b200_trisolve* p, double* d_x, cudaStream_t s) {
    sprs_b200_ctx* ctx = p->ctx;
    SPRS_TRY(take_breach(p, "in an earlier solve_dev of this plan"));
    if (++p->epoch == 0) {
        SPRS_CUDA(ctx, cudaMemsetAsync(p->d_flags, 0, p->n * sizeof(uint32_t), s));
        p->epoch = 1;
    }
    SPRS_TRY(p->csr->indptr_bytes == 4 ? launch_solve<uint32_t>(p, d_x, s)
                                       : launch_solve<uint64_t>(p, d_x, s));
    SPRS_CUDA(ctx, cudaEventRecord(p->ev_last, s));
    return SPRS_B200_OK;
}

int singular_status(sprs_b200_trisolve* p) {
    if (p->k_ticket >= p->n) return SPRS_B200_OK;
    static const char* reasons[] = {"diagonal element is 0", "diagonal element is a numeric 0",
                                    "diagonal element is a structural 0"};
    SPRS_FAIL(p->ctx, SPRS_B200_ERR_SINGULAR, "Singular matrix at index %llu (%s)",
              (unsigned long long)p->sing_index, reasons[p->sing_reason]);
}

void free_plan(sprs_b200_trisolve* p) {
    if (p->ctx) cudaSetDevice(p->ctx->device);
    if (p->d_diag) cudaFree(p->d_diag);
    if (p->d_flags) cudaFree(p->d_flags);
    if (p->d_words) cudaFree(p->d_words);
    if (p->d_progress) cudaFree(p->d_progress);
    if (p->h_err) cudaFreeHost(p->h_err);
    if (p->ev_last) cudaEventDestroy(p->ev_last);
    if (p->own_t) sprs_b200_csmat_free(p->own_t);
    delete p;
}

// the flags, counters and wait-bound words of a plan
int alloc_solve_state(sprs_b200_trisolve* p, cudaStream_t s) {
    sprs_b200_ctx* ctx = p->ctx;
    const uint64_t n = p->n;
    SPRS_CUDA(ctx, cudaMalloc((void**)&p->d_flags, n * sizeof(uint32_t) + 16));
    SPRS_CUDA(ctx, cudaMalloc((void**)&p->d_words, 2 * sizeof(unsigned long long)));
    p->n_progress = (uint64_t)ctx->sm_count * TRI_CTAS_PER_SM * (TRI_THREADS / 32);
    SPRS_CUDA(ctx, cudaMalloc((void**)&p->d_progress, p->n_progress * sizeof(unsigned long long)));
    SPRS_CUDA(ctx, cudaEventCreateWithFlags(&p->ev_last, cudaEventDisableTiming));
    SPRS_CUDA(ctx, cudaMallocHost((void**)&p->h_err, sizeof(unsigned long long)));
    *p->h_err = 0;
    SPRS_CUDA(ctx, cudaMemsetAsync(p->d_flags, 0, n * sizeof(uint32_t) + 16, s));
    return SPRS_B200_OK;
}

int build_plan(sprs_b200_trisolve* p, const sprs_b200_csmat* mat) {
    sprs_b200_ctx* ctx = p->ctx;
    cudaStream_t s = ctx->stream;
    if (mat->storage == SPRS_B200_CSC) {
        p->own_t = new sprs_b200_csmat();
        SPRS_TRY(transpose_launch(ctx, mat, p->own_t, s));
        p->csr = p->own_t;
    } else {
        p->csr = mat;
    }
    const uint64_t n = p->n;
    SPRS_CUDA(ctx, cudaMalloc((void**)&p->d_diag, n * sizeof(uint32_t) + 16));
    SPRS_TRY(alloc_solve_state(p, s));
    unsigned long long key = ~0ull;
    SPRS_CUDA(ctx, cudaMemcpyAsync(p->d_words + 1, &key, sizeof(key), cudaMemcpyHostToDevice, s));
    if (n) SPRS_TRY(p->csr->indptr_bytes == 4 ? launch_plan<uint32_t>(p, s) : launch_plan<uint64_t>(p, s));
    SPRS_CUDA(ctx, cudaMemcpyAsync(&key, p->d_words + 1, sizeof(key), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    p->k_ticket = n;
    if (key != ~0ull) {
        const bool present = key & 1;
        p->k_ticket = key >> 1;
        p->sing_index = p->tri == SPRS_B200_TRI_UPPER ? n - 1 - p->k_ticket : p->k_ticket;
        if (p->storage == SPRS_B200_CSC)
            p->sing_reason = present ? SPRS_B200_SINGULAR_NUMERIC : SPRS_B200_SINGULAR_STRUCTURAL;
        else
            p->sing_reason = p->tri == SPRS_B200_TRI_LOWER ? SPRS_B200_SINGULAR_IS_ZERO
                                                           : SPRS_B200_SINGULAR_NUMERIC;
    }
    return SPRS_B200_OK;
}

}  // namespace

int trisolve_unit_plan(sprs_b200_ctx* ctx, const sprs_b200_csmat* csr, int tri,
                       sprs_b200_trisolve** out) {
    *out = nullptr;
    auto* p = new sprs_b200_trisolve();
    p->ctx = ctx;
    p->csr = csr;
    p->tri = tri;
    p->n = csr->rows;
    p->k_ticket = p->n;
    p->unit = true;
    const int st = alloc_solve_state(p, ctx->stream);
    if (st != SPRS_B200_OK) {
        free_plan(p);
        return st;
    }
    *out = p;
    return SPRS_B200_OK;
}

int trisolve_enqueue(sprs_b200_trisolve* plan, double* d_x, cudaStream_t s) {
    return enqueue_solve(plan, d_x, s);
}

int trisolve_check_breach(sprs_b200_trisolve* plan) {
    return take_breach(plan, "in this solve");
}

extern "C" {

int sprs_b200_trisolve_plan(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, int tri,
                            sprs_b200_trisolve** out) {
    if (!ctx || !mat || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if (tri != SPRS_B200_TRI_LOWER && tri != SPRS_B200_TRI_UPPER)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "trisolve: unknown triangle %d", tri);
    if (mat->rows != mat->cols)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Non square matrix passed to solver");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    auto* p = new sprs_b200_trisolve();
    p->ctx = ctx;
    p->storage = mat->storage;
    p->tri = tri;
    p->n = mat->rows;
    const int st = build_plan(p, mat);
    if (st != SPRS_B200_OK) {
        free_plan(p);
        return st;
    }
    *out = p;
    return SPRS_B200_OK;
}

int sprs_b200_trisolve_singular(const sprs_b200_trisolve* plan, uint64_t* index, int* reason) {
    if (!plan) return 0;
    const bool sing = plan->k_ticket < plan->n;
    if (sing && index) *index = plan->sing_index;
    if (sing && reason) *reason = plan->sing_reason;
    return sing ? 1 : 0;
}

int sprs_b200_trisolve_solve(sprs_b200_trisolve* plan, double* rhs, uint64_t len) {
    if (!plan) return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_ctx* ctx = plan->ctx;
    if (len != plan->n) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (len && !rhs) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    void* d_x = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 1, len * sizeof(double), &d_x));
    if (len)
        SPRS_CUDA(ctx, cudaMemcpyAsync(d_x, rhs, len * sizeof(double), cudaMemcpyHostToDevice, s));
    SPRS_TRY(enqueue_solve(plan, (double*)d_x, s));
    if (len)
        SPRS_CUDA(ctx, cudaMemcpyAsync(rhs, d_x, len * sizeof(double), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    SPRS_TRY(take_breach(plan, "in this solve"));
    return singular_status(plan);
}

int sprs_b200_trisolve_solve_dev(sprs_b200_trisolve* plan, double* d_rhs, void* stream) {
    if (!plan || (plan->n && !d_rhs)) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(plan->ctx, cudaSetDevice(plan->ctx->device));
    SPRS_TRY(enqueue_solve(plan, d_rhs, pick_stream(plan->ctx, stream)));
    return singular_status(plan);
}

int sprs_b200_trisolve_free(sprs_b200_trisolve* plan) {
    if (!plan) return SPRS_B200_OK;
    cudaSetDevice(plan->ctx->device);
    // the last solve_dev, on whatever stream it was enqueued, may still use the plan
    cudaStreamWaitEvent(plan->ctx->stream, plan->ev_last, 0);
    cudaStreamSynchronize(plan->ctx->stream);
    free_plan(plan);
    return SPRS_B200_OK;
}

}  // extern "C"
