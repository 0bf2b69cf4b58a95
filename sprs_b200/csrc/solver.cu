// solver.cu -- device-resident BiCGSTAB, the iterative caller of the SpMV path
// (SURVEY.md 8f rank 3; reference: sprs/src/sparse/linalg/bicgstab.rs:95-300).
//
// Every vector of the iteration (x, r, rhat, p and the temporaries v, s, t) lives in HBM for
// the whole solve; only three pairs of scalars per step cross PCIe (16 B each).  The matrix
// products are the library's SpMV (spmv.cu); the vector algebra of one step is fused into
// five streaming kernels:
//     v = A p                                        spmv
//     d1 = rhat.v                                    dot2_kernel        -> alpha = rho / d1
//     s = r - v*alpha                                s_kernel
//     t = A s                                        spmv
//     (t.s, t.t)                                     dot2_kernel        -> omega
//     x = (x + p*alpha) + omega*s ; r = s - t*omega ; (r.r, rhat.r)   update_kernel
//     p = r + (p - v*omega)*beta   |   rhat = p = r (soft restart)    p_kernel | copy2_kernel
// Arithmetic follows the reference operation by operation (product rounded, then the sum or
// difference rounded: __dmul_rn / __dadd_rn / __dsub_rn, never an FMA); the scalar algebra
// (alpha, omega, beta, the restart test) runs on the host in the reference's order.
//
// Reductions are deterministic: a thread sums its elements sequentially in index order, in
// chunks of 4 consecutive elements, then a fixed shuffle/shared-memory tree combines the
// threads and a second one-block kernel combines the blocks.  The reference sums strictly
// sequentially (vec.rs:846-881, 907-913), so results agree to rounding, and exactly when
// n <= 4 (one thread holds the whole sum; adding the other threads' +0.0 changes nothing).
// HBM-bound: 16 vector passes (128 B per row) per step next to 2 SpMVs.
#include <cmath>

#include "common.cuh"

namespace {

constexpr int RED_THREADS = 256;
constexpr int RED_MAX_BLOCKS = 1024;  // partial sums per reduction (two doubles each)

__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

// Fixed-order block reduction of two running sums; thread 0 writes partials[2*block + {0,1}].
__device__ __forceinline__ void block_reduce2(double s0, double s1, double* partials) {
    __shared__ double sh[2][RED_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s0 = add_rn(s0, __shfl_down_sync(0xffffffffu, s0, o));
        s1 = add_rn(s1, __shfl_down_sync(0xffffffffu, s1, o));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        sh[0][warp] = s0;
        sh[1][warp] = s1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = sh[0][0], b = sh[1][0];
        for (int w = 1; w < RED_THREADS / 32; ++w) {
            a = add_rn(a, sh[0][w]);
            b = add_rn(b, sh[1][w]);
        }
        partials[2 * blockIdx.x] = a;
        partials[2 * blockIdx.x + 1] = b;
    }
}

// One block: out[j] = sum over blocks of partials[2*b + j], fixed order.
__global__ void __launch_bounds__(RED_THREADS) final_reduce_kernel(const double* partials,
                                                                   int n_blocks, double* out) {
    double s0 = 0.0, s1 = 0.0;
    for (int b = threadIdx.x; b < n_blocks; b += RED_THREADS) {
        s0 = add_rn(s0, partials[2 * b]);
        s1 = add_rn(s1, partials[2 * b + 1]);
    }
    // block_reduce2 writes to partials[2*blockIdx.x..]: blockIdx.x == 0, so `out` directly
    block_reduce2(s0, s1, out);
}

// Chunked grid-stride loop: chunk c covers elements [4c, 4c+4); a thread visits chunks
// tid, tid + nthreads, ... in increasing order.  All vectors are the solver's own buffers
// (256-byte aligned), so a full chunk moves as two 16-byte accesses per vector.
#define FOR_EACH_CHUNK(n)                                                                  \
    for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x,                     \
                  stride = (uint64_t)gridDim.x * blockDim.x, nchunks = ((n) + 3) / 4;      \
         c < nchunks; c += stride)

struct Chunk {
    double v[4];
};
__device__ __forceinline__ Chunk load_chunk(const double* p, uint64_t i0, int cnt) {
    Chunk r;
    if (cnt == 4) {
        const double2 a = *reinterpret_cast<const double2*>(p + i0);
        const double2 b = *reinterpret_cast<const double2*>(p + i0 + 2);
        r.v[0] = a.x, r.v[1] = a.y, r.v[2] = b.x, r.v[3] = b.y;
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) r.v[k] = k < cnt ? p[i0 + k] : 0.0;
    }
    return r;
}
__device__ __forceinline__ void store_chunk(double* p, uint64_t i0, int cnt, const Chunk& r) {
    if (cnt == 4) {
        *reinterpret_cast<double2*>(p + i0) = make_double2(r.v[0], r.v[1]);
        *reinterpret_cast<double2*>(p + i0 + 2) = make_double2(r.v[2], r.v[3]);
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (k < cnt) p[i0 + k] = r.v[k];
    }
}
#define CHUNK_BOUNDS(n)          \
    const uint64_t i0 = 4 * c;   \
    const int cnt = (n) - i0 < 4 ? (int)((n) - i0) : 4

// (a1.b1, a2.b2); a2 == nullptr computes only the first.
__global__ void __launch_bounds__(RED_THREADS)
    dot2_kernel(const double* __restrict__ a1, const double* __restrict__ b1,
                const double* a2, const double* b2, uint64_t n, double* partials) {
    double s0 = 0.0, s1 = 0.0;
    FOR_EACH_CHUNK(n) {
        CHUNK_BOUNDS(n);
        const Chunk x1 = load_chunk(a1, i0, cnt), y1 = load_chunk(b1, i0, cnt);
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (k < cnt) s0 = add_rn(s0, mul_rn(x1.v[k], y1.v[k]));
        if (a2) {
            const Chunk x2 = load_chunk(a2, i0, cnt), y2 = load_chunk(b2, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (k < cnt) s1 = add_rn(s1, mul_rn(x2.v[k], y2.v[k]));
        }
    }
    block_reduce2(s0, s1, partials);
}

// r = b - ax ; rhat = r ; p = r ; partial r.r            (bicgstab.rs:125-129, 186-196)
__global__ void __launch_bounds__(RED_THREADS)
    residual_kernel(const double* __restrict__ b, const double* __restrict__ ax,
                    double* __restrict__ r, double* __restrict__ rhat, double* __restrict__ p,
                    uint64_t n, double* partials) {
    double s0 = 0.0;
    FOR_EACH_CHUNK(n) {
        CHUNK_BOUNDS(n);
        const Chunk bv = load_chunk(b, i0, cnt), av = load_chunk(ax, i0, cnt);
        Chunk rv;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            rv.v[k] = sub_rn(bv.v[k], av.v[k]);
            if (k < cnt) s0 = add_rn(s0, mul_rn(rv.v[k], rv.v[k]));
        }
        store_chunk(r, i0, cnt, rv);
        store_chunk(rhat, i0, cnt, rv);
        store_chunk(p, i0, cnt, rv);
    }
    block_reduce2(s0, 0.0, partials);
}

// s = r - v*alpha                                         (bicgstab.rs:207)
__global__ void __launch_bounds__(RED_THREADS)
    s_kernel(const double* __restrict__ r, const double* __restrict__ v, double alpha,
             double* __restrict__ s, uint64_t n) {
    FOR_EACH_CHUNK(n) {
        CHUNK_BOUNDS(n);
        const Chunk rv = load_chunk(r, i0, cnt), vv = load_chunk(v, i0, cnt);
        Chunk sv;
#pragma unroll
        for (int k = 0; k < 4; ++k) sv.v[k] = sub_rn(rv.v[k], mul_rn(vv.v[k], alpha));
        store_chunk(s, i0, cnt, sv);
    }
}

// x = (x + p*alpha) + omega*s ; r = s - t*omega ; partial (r.r, rhat.r)
//                                                         (bicgstab.rs:204, 210, 213-218)
__global__ void __launch_bounds__(RED_THREADS)
    update_kernel(double* x, const double* __restrict__ p, const double* __restrict__ s,
                  const double* __restrict__ t, const double* __restrict__ rhat, double alpha,
                  double omega, double* __restrict__ r, uint64_t n, double* partials) {
    double s0 = 0.0, s1 = 0.0;
    FOR_EACH_CHUNK(n) {
        CHUNK_BOUNDS(n);
        const Chunk xv = load_chunk(x, i0, cnt), pv = load_chunk(p, i0, cnt),
                    sv = load_chunk(s, i0, cnt), tv = load_chunk(t, i0, cnt),
                    hv = load_chunk(rhat, i0, cnt);
        Chunk xn, rn;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const double h = add_rn(xv.v[k], mul_rn(pv.v[k], alpha));
            xn.v[k] = add_rn(h, mul_rn(omega, sv.v[k]));
            rn.v[k] = sub_rn(sv.v[k], mul_rn(tv.v[k], omega));
            if (k < cnt) {
                s0 = add_rn(s0, mul_rn(rn.v[k], rn.v[k]));
                s1 = add_rn(s1, mul_rn(hv.v[k], rn.v[k]));
            }
        }
        store_chunk(x, i0, cnt, xn);
        store_chunk(r, i0, cnt, rn);
    }
    block_reduce2(s0, s1, partials);
}

// p = r + (p - v*omega)*beta                              (bicgstab.rs:227-229)
__global__ void __launch_bounds__(RED_THREADS)
    p_kernel(const double* __restrict__ r, const double* __restrict__ v, double omega,
             double beta, double* p, uint64_t n) {
    FOR_EACH_CHUNK(n) {
        CHUNK_BOUNDS(n);
        const Chunk rv = load_chunk(r, i0, cnt), vv = load_chunk(v, i0, cnt),
                    pv = load_chunk(p, i0, cnt);
        Chunk pn;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            pn.v[k] = add_rn(rv.v[k], mul_rn(sub_rn(pv.v[k], mul_rn(vv.v[k], omega)), beta));
        store_chunk(p, i0, cnt, pn);
    }
}

// rhat = r ; p = r                                        (bicgstab.rs:179-183)
__global__ void __launch_bounds__(RED_THREADS)
    copy2_kernel(const double* __restrict__ r, double* __restrict__ rhat,
                 double* __restrict__ p, uint64_t n) {
    FOR_EACH_CHUNK(n) {
        CHUNK_BOUNDS(n);
        const Chunk rv = load_chunk(r, i0, cnt);
        store_chunk(rhat, i0, cnt, rv);
        store_chunk(p, i0, cnt, rv);
    }
}

}  // namespace

struct sprs_b200_bicgstab {
    sprs_b200_ctx* ctx = nullptr;
    const sprs_b200_csmat* csr = nullptr;  // borrowed (the operand, or its cached CSR form)
    // operator form (sprs_b200_bicgstab_new_op): y = A x is the caller's, e.g. the
    // row-partitioned SpMV + all-gather of sprs_b200/dist.py; csr stays null
    sprs_b200_matvec_fn op = nullptr;
    void* op_user = nullptr;
    uint64_t n = 0;
    Owned<double> d_block;      // one allocation: 8 vectors of `pitch` doubles
    uint64_t pitch = 0;
    double *d_b = nullptr, *d_x = nullptr, *d_r = nullptr, *d_rhat = nullptr, *d_p = nullptr,
           *d_v = nullptr, *d_s = nullptr, *d_t = nullptr;
    Owned<double> d_partials;      // 2 * RED_MAX_BLOCKS, then the 2 results
    Owned<double> h_result;        // pinned, 2 doubles
    int grid = 1;
    // bicgstab.rs:97-116
    uint64_t iteration_count = 0, soft_restart_count = 0, hard_restart_count = 0;
    double soft_restart_threshold = 0.1;
    double err = 0.0, rho = 0.0;
};

namespace {

// finish a reduction started by a kernel that wrote `grid` partial pairs: results in
// h_result[0..1] once this returns (one 16-byte D2H copy + stream sync).
int finish_reduce(sprs_b200_bicgstab* s, cudaStream_t st) {
    sprs_b200_ctx* ctx = s->ctx;
    if (s->n == 0) {
        s->h_result[0] = s->h_result[1] = 0.0;  // empty sums (Rust's Sum of nothing)
        return SPRS_B200_OK;
    }
    double* d_out = s->d_partials + 2 * RED_MAX_BLOCKS;
    final_reduce_kernel<<<1, RED_THREADS, 0, st>>>(s->d_partials, s->grid, d_out);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    SPRS_CUDA(ctx, cudaMemcpyAsync(s->h_result, d_out, 2 * sizeof(double),
                                   cudaMemcpyDeviceToHost, st));
    SPRS_CUDA(ctx, cudaStreamSynchronize(st));
    return SPRS_B200_OK;
}

// y = A x  (`&a * &x`: a fresh zero vector is accumulated into, csmat.rs:2119-2160)
int matvec(sprs_b200_bicgstab* s, const double* d_x, double* d_y, cudaStream_t st) {
    if (s->n == 0) return SPRS_B200_OK;
    if (s->op) {
        if (s->op(s->op_user, d_x, d_y, (void*)st) != 0)
            SPRS_FAIL(s->ctx, SPRS_B200_ERR_ARGUMENT, "bicgstab: the matvec callback failed");
        return SPRS_B200_OK;
    }
    return spmv_launch(s->ctx, s->csr, d_x, d_y, /*accumulate=*/0, st);
}

// r = b - A x ; rhat = p = r ; err = |r| ; rho = err^2 (new(), and hard_restart's recompute)
int recompute_residual(sprs_b200_bicgstab* s) {
    sprs_b200_ctx* ctx = s->ctx;
    cudaStream_t st = ctx->stream;
    SPRS_TRY(matvec(s, s->d_x, s->d_v, st));
    if (s->n) {
        residual_kernel<<<s->grid, RED_THREADS, 0, st>>>(s->d_b, s->d_v, s->d_r, s->d_rhat,
                                                         s->d_p, s->n, s->d_partials);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaGetLastError());
    }
    SPRS_TRY(finish_reduce(s, st));
    s->err = std::sqrt(s->h_result[0]);
    s->rho = s->err * s->err;
    return SPRS_B200_OK;
}

int create_common(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, sprs_b200_matvec_fn op,
                  void* op_user, const double* x0, const double* b, uint64_t n,
                  cudaMemcpyKind kind, sprs_b200_bicgstab** out) {
    if (!ctx || (!mat && !op) || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    // `&a * &x0` and `&b - &(..)` panic on mismatched dimensions (prod.rs:170, binop.rs:455);
    // A p with p = r needs a square matrix
    if (mat && (mat->rows != n || mat->cols != n))
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (n && (!x0 || !b)) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    const sprs_b200_csmat* csr = nullptr;
    if (mat) SPRS_TRY(csmat_csr_view(ctx, mat, &csr));
    std::unique_ptr<sprs_b200_bicgstab, FreeWith<sprs_b200_bicgstab_free>> s(
        new sprs_b200_bicgstab());
    s->ctx = ctx;
    s->csr = csr;
    s->op = mat ? nullptr : op;
    s->op_user = op_user;
    s->n = n;
    s->pitch = (n + 31) / 32 * 32 + 32;  // 256-byte aligned vectors
    SPRS_TRY(s->d_block.alloc(ctx, 8 * s->pitch * sizeof(double), "bicgstab"));
    SPRS_TRY(s->d_partials.alloc(ctx, (2 * RED_MAX_BLOCKS + 2) * sizeof(double), "bicgstab"));
    SPRS_TRY(s->h_result.alloc_pinned(ctx, 2 * sizeof(double), "bicgstab"));
    double** slots[8] = {&s->d_b, &s->d_x, &s->d_r, &s->d_rhat,
                         &s->d_p, &s->d_v, &s->d_s, &s->d_t};
    for (int i = 0; i < 8; ++i) *slots[i] = s->d_block + (uint64_t)i * s->pitch;
    uint64_t blocks = (n + 4 * RED_THREADS - 1) / (4 * RED_THREADS);
    if (blocks < 1) blocks = 1;
    const uint64_t cap = (uint64_t)ctx->sm_count * 4 < RED_MAX_BLOCKS
                             ? (uint64_t)ctx->sm_count * 4
                             : RED_MAX_BLOCKS;
    s->grid = (int)(blocks < cap ? blocks : cap);
    if (n) {
        cudaStream_t cs = ctx->stream;
        SPRS_CUDA(ctx, cudaMemcpyAsync(s->d_x, x0, n * sizeof(double), kind, cs));
        SPRS_CUDA(ctx, cudaMemcpyAsync(s->d_b, b, n * sizeof(double), kind, cs));
    }
    SPRS_TRY(recompute_residual(s.get()));  // synchronises the stream: x0 / b may be reused after
    *out = s.release();
    return SPRS_B200_OK;
}

}  // namespace

int sprs_b200_bicgstab_new(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* x0,
                           const double* b, uint64_t n, sprs_b200_bicgstab** out) {
    return create_common(ctx, mat, nullptr, nullptr, x0, b, n, cudaMemcpyHostToDevice, out);
}

int sprs_b200_bicgstab_new_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                               const double* d_x0, const double* d_b, uint64_t n,
                               sprs_b200_bicgstab** out) {
    return create_common(ctx, mat, nullptr, nullptr, d_x0, d_b, n, cudaMemcpyDeviceToDevice, out);
}

int sprs_b200_bicgstab_new_op(sprs_b200_ctx* ctx, uint64_t n, sprs_b200_matvec_fn matvec,
                              void* user, const double* x0, const double* b,
                              int device_pointers, sprs_b200_bicgstab** out) {
    if (!matvec) return SPRS_B200_ERR_ARGUMENT;
    return create_common(ctx, nullptr, matvec, user, x0, b, n,
                         device_pointers ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, out);
}

int sprs_b200_bicgstab_free(sprs_b200_bicgstab* s) {
    if (!s) return SPRS_B200_OK;
    if (s->ctx) cudaSetDevice(s->ctx->device);
    delete s;
    return SPRS_B200_OK;
}

// bicgstab.rs:177-184
int sprs_b200_bicgstab_soft_restart(sprs_b200_bicgstab* s) {
    if (!s) return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_ctx* ctx = s->ctx;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    s->soft_restart_count += 1;
    s->rho = s->err * s->err;
    if (s->n) {
        copy2_kernel<<<s->grid, RED_THREADS, 0, ctx->stream>>>(s->d_r, s->d_rhat, s->d_p, s->n);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaGetLastError());
    }
    return SPRS_B200_OK;
}

// bicgstab.rs:186-196 (the copies rhat = p = r ride in the residual kernel)
int sprs_b200_bicgstab_hard_restart(sprs_b200_bicgstab* s) {
    if (!s) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(s->ctx, cudaSetDevice(s->ctx->device));
    s->hard_restart_count += 1;
    return recompute_residual(s);
}

// bicgstab.rs:198-234
int sprs_b200_bicgstab_step(sprs_b200_bicgstab* s, double* err_out) {
    if (!s) return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_ctx* ctx = s->ctx;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const uint64_t n = s->n;
    s->iteration_count += 1;

    // gradient descent step
    SPRS_TRY(matvec(s, s->d_p, s->d_v, st));
    if (n) {
        dot2_kernel<<<s->grid, RED_THREADS, 0, st>>>(s->d_rhat, s->d_v, nullptr, nullptr, n,
                                                     s->d_partials);
        ctx->launches += 1;
    }
    SPRS_TRY(finish_reduce(s, st));
    const double alpha = s->rho / s->h_result[0];

    // conjugate direction step
    if (n) {
        s_kernel<<<s->grid, RED_THREADS, 0, st>>>(s->d_r, s->d_v, alpha, s->d_s, n);
        ctx->launches += 1;
    }
    SPRS_TRY(matvec(s, s->d_s, s->d_t, st));
    if (n) {
        dot2_kernel<<<s->grid, RED_THREADS, 0, st>>>(s->d_t, s->d_s, s->d_t, s->d_t, n,
                                                     s->d_partials);
        ctx->launches += 1;
    }
    SPRS_TRY(finish_reduce(s, st));
    const double omega = s->h_result[0] / s->h_result[1];

    // new x, new r, error
    if (n) {
        update_kernel<<<s->grid, RED_THREADS, 0, st>>>(s->d_x, s->d_p, s->d_s, s->d_t, s->d_rhat,
                                                       alpha, omega, s->d_r, n, s->d_partials);
        ctx->launches += 1;
    }
    SPRS_TRY(finish_reduce(s, st));
    s->err = std::sqrt(s->h_result[0]);
    const double rho_prev = s->rho;
    s->rho = s->h_result[1];

    // soft restart if rhat is becoming perpendicular to r
    if (std::fabs(s->rho) / (s->err * s->err) < s->soft_restart_threshold) {
        SPRS_TRY(sprs_b200_bicgstab_soft_restart(s));
    } else {
        const double beta = (s->rho / rho_prev) * (alpha / omega);
        if (n) {
            p_kernel<<<s->grid, RED_THREADS, 0, st>>>(s->d_r, s->d_v, omega, beta, s->d_p, n);
            ctx->launches += 1;
        }
    }
    SPRS_CUDA(ctx, cudaGetLastError());
    if (err_out) *err_out = s->err;
    return SPRS_B200_OK;
}

// bicgstab.rs:151-175: *converged = 1 for Ok, 0 for Err; the state is kept either way
int sprs_b200_bicgstab_solve(sprs_b200_bicgstab* s, double tol, uint64_t max_iter,
                             int* converged) {
    if (!s || !converged) return SPRS_B200_ERR_ARGUMENT;
    *converged = 0;
    for (uint64_t it = 0; it < max_iter; ++it) {
        SPRS_TRY(sprs_b200_bicgstab_step(s, nullptr));
        if (s->err < tol) {
            // check the true error before claiming convergence
            SPRS_TRY(sprs_b200_bicgstab_hard_restart(s));
            if (s->err < tol) {
                *converged = 1;
                break;
            }
        }
    }
    // queued vector updates (p) finish before the caller looks at the state
    SPRS_CUDA(s->ctx, cudaStreamSynchronize(s->ctx->stream));
    return SPRS_B200_OK;
}

int sprs_b200_bicgstab_set_restart_threshold(sprs_b200_bicgstab* s, double thresh) {
    if (!s) return SPRS_B200_ERR_ARGUMENT;
    s->soft_restart_threshold = thresh;
    return SPRS_B200_OK;
}

int sprs_b200_bicgstab_stats(const sprs_b200_bicgstab* s, uint64_t counts[3],
                             double scalars[3]) {
    if (!s) return SPRS_B200_ERR_ARGUMENT;
    if (counts) {
        counts[0] = s->iteration_count;
        counts[1] = s->soft_restart_count;
        counts[2] = s->hard_restart_count;
    }
    if (scalars) {
        scalars[0] = s->err;
        scalars[1] = s->rho;
        scalars[2] = s->soft_restart_threshold;
    }
    return SPRS_B200_OK;
}

static double* vector_of(const sprs_b200_bicgstab* s, int which) {
    switch (which) {
        case SPRS_B200_BICGSTAB_X: return s->d_x;
        case SPRS_B200_BICGSTAB_R: return s->d_r;
        case SPRS_B200_BICGSTAB_RHAT: return s->d_rhat;
        case SPRS_B200_BICGSTAB_P: return s->d_p;
        case SPRS_B200_BICGSTAB_B: return s->d_b;
        default: return nullptr;
    }
}

int sprs_b200_bicgstab_get(const sprs_b200_bicgstab* s, int which, double* out, uint64_t len) {
    if (!s) return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_ctx* ctx = s->ctx;
    const double* d = vector_of(s, which);
    if (!d) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "bicgstab_get: unknown vector id %d", which);
    if (len != s->n) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (!len) return SPRS_B200_OK;
    if (!out) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    SPRS_CUDA(ctx, cudaMemcpyAsync(out, d, len * sizeof(double), cudaMemcpyDeviceToHost,
                                   ctx->stream));
    SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SPRS_B200_OK;
}

int sprs_b200_bicgstab_get_dev(const sprs_b200_bicgstab* s, int which, const double** d_out) {
    if (!s || !d_out) return SPRS_B200_ERR_ARGUMENT;
    *d_out = vector_of(s, which);
    if (!*d_out) SPRS_FAIL(s->ctx, SPRS_B200_ERR_ARGUMENT, "bicgstab_get_dev: unknown vector id");
    // work queued on the library's stream is complete before the caller's stream reads
    SPRS_CUDA(s->ctx, cudaSetDevice(s->ctx->device));
    SPRS_CUDA(s->ctx, cudaStreamSynchronize(s->ctx->stream));
    return SPRS_B200_OK;
}
