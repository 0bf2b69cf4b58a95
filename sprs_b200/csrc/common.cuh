// common.cuh -- internal types shared by the sm_90a kernels and the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/sprs_b200.h"

constexpr int SPRS_E2E_MAX_CHUNKS = 8;
constexpr int SPRS_E2E_DEFAULT_CHUNKS = 8;  // host path: y leaves in 8 chunks behind the SpMV
                                            // (1 = one launch + one copy)

// ---- error plumbing: C functions return int, never throw/abort (SURVEY 8b) ----
struct sprs_b200_ctx {
    int device = 0;
    int sm_count = 132;
    size_t l2_bytes = 0;
    cudaStream_t stream = nullptr;  // private stream of the host-buffer entry points
    std::string last_error;
    uint64_t launches = 0;
    // L2 cache-policy words (createpolicy results), produced once per ctx: kernels take them as
    // parameters so that they live in uniform registers
    uint64_t pol_evict_first = 0, pol_evict_last = 0;
    // pinned host staging + device scratch for the host-buffer entry points
    void* h_stage = nullptr;
    size_t h_stage_bytes = 0;
    void* d_scratch[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t d_scratch_bytes[4] = {0, 0, 0, 0};
    // chunked push (peer.cu): high-priority side stream of the put kernels and the fork/join
    // events that tie it to the caller's stream; created on first use
    cudaStream_t side_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // chunked host path (api.cu, SPRS_B200_E2E_PIPELINE=2): copy stream + one event per chunk
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_chunk[SPRS_E2E_MAX_CHUNKS] = {};
    cudaEvent_t ev_copied = nullptr;
};

struct sprs_b200_csmat {
    sprs_b200_ctx* ctx = nullptr;
    int storage = SPRS_B200_CSR;
    uint64_t rows = 0, cols = 0, nnz = 0;
    uint64_t outer = 0, inner = 0;
    int indptr_bytes = 4;          // 4 unless nnz >= 2^32
    void* d_indptr = nullptr;      // outer+1 entries
    uint32_t* d_indices = nullptr; // nnz entries
    double* d_data = nullptr;      // nnz entries
    bool owns = true;              // false for from_device adoption
    bool pooled = false;           // arrays came from cudaMallocAsync (SpGEMM results)
    // SpMV partition (spmv.cu): merge-path cuts (tile_row[t], tile_k[t]) = rows passed / nnz
    // consumed at cost t*W; n_tiles+1 entries each.  carry: n_tiles doubles.
    uint32_t* d_tile_row = nullptr;
    void* d_tile_k = nullptr;      // nnz position of every cut (as wide as the indptr)
    double* d_carry = nullptr;
    uint64_t n_tiles = 0;
    // SpMV hot set (spmv.cu, DESIGN.md 4.1): the n_hot most-referenced columns (hot_col, K
    // entries) and the index stream the SpMV reads instead of d_indices, each hot column tagged
    // as 0x80000000 | slot (hot_idx, nnz entries: +4 bytes per non-zero).  n_hot == 0: none.
    uint32_t* d_hot_col = nullptr;
    uint32_t* d_hot_idx = nullptr;
    uint32_t n_hot = 0;
    // CSC mirrors only: the CSR conversion the product kernels run on, built on first use
    // by the host-buffer entry points and kept until the mirror is freed.
    mutable sprs_b200_csmat* csr_cache = nullptr;
    // chunked host path only: tile and row boundaries of the chunks (host copies, built on
    // first use: chunk c covers tiles [e2e_tiles[c], e2e_tiles[c+1]) and completes rows
    // [e2e_rows[c], e2e_rows[c+1]))
    mutable std::vector<uint64_t> e2e_tiles, e2e_rows;
    // chunked push (peer.cu): the same kind of table with front-loaded chunk sizes
    mutable std::vector<uint64_t> push_tiles, push_rows;
};

#define SPRS_FAIL(ctx, code, ...)                                  \
    do {                                                           \
        char _buf[512];                                            \
        snprintf(_buf, sizeof(_buf), __VA_ARGS__);                 \
        sprs_b200_set_error((ctx), _buf);                          \
        return (code);                                             \
    } while (0)

#define SPRS_CUDA(ctx, expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess)                                                            \
            SPRS_FAIL((ctx), SPRS_B200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,          \
                      cudaGetErrorString(_e), __FILE__, __LINE__);                        \
    } while (0)

#define SPRS_TRY(expr)                      \
    do {                                    \
        int _s = (expr);                    \
        if (_s != SPRS_B200_OK) return _s;  \
    } while (0)

void sprs_b200_set_error(const sprs_b200_ctx* ctx, const char* msg);

// Device-resident entry points run on exactly the stream they are given; NULL is the
// CUDA legacy default stream (that is what torch's default stream is), NOT ctx->stream.
static inline cudaStream_t pick_stream(sprs_b200_ctx*, void* stream) {
    return (cudaStream_t)stream;
}

// scratch slot `i` of at least `bytes` (grown geometrically, contents undefined)
int ctx_scratch(sprs_b200_ctx* ctx, int i, size_t bytes, void** out);
int ctx_stage(sprs_b200_ctx* ctx, size_t bytes, void** out);

// ---- scoped ownership (host code) -----------------------------------------------
// Where an owned allocation comes from: cudaMalloc, cudaMallocAsync (freed on the stream it was
// allocated on) or cudaMallocHost.
enum class MemKind { device, stream, pinned };
// `bytes` of `kind` into *p.  On failure: clears the runtime's error, sets the ctx's last error
// to "<what>: ..." and returns ERR_CUDA (api.cu).
int mem_alloc(sprs_b200_ctx* ctx, MemKind kind, size_t bytes, cudaStream_t s, const char* what,
              void** p);
void mem_free(MemKind kind, void* p, cudaStream_t s);

// One allocation, released when its owner goes out of scope (or on reset / the next alloc).
template <typename T>
class Owned {
  public:
    Owned() = default;
    Owned(const Owned&) = delete;
    Owned& operator=(const Owned&) = delete;
    Owned(Owned&& o) noexcept : p_(o.release()), kind_(o.kind_), s_(o.s_) {}
    ~Owned() { reset(); }

    int alloc(sprs_b200_ctx* ctx, size_t bytes, const char* what) {
        return take(ctx, MemKind::device, bytes, nullptr, what);
    }
    int alloc_async(sprs_b200_ctx* ctx, size_t bytes, cudaStream_t s, const char* what) {
        return take(ctx, MemKind::stream, bytes, s, what);
    }
    int alloc_pinned(sprs_b200_ctx* ctx, size_t bytes, const char* what) {
        return take(ctx, MemKind::pinned, bytes, nullptr, what);
    }
    void reset() {
        if (p_) mem_free(kind_, p_, s_);
        p_ = nullptr;
    }
    T* release() {
        T* p = p_;
        p_ = nullptr;
        return p;
    }
    operator T*() const { return p_; }

  private:
    int take(sprs_b200_ctx* ctx, MemKind kind, size_t bytes, cudaStream_t s, const char* what) {
        reset();
        void* p = nullptr;
        SPRS_TRY(mem_alloc(ctx, kind, bytes, s, what, &p));
        p_ = (T*)p;
        kind_ = kind;
        s_ = s;
        return SPRS_B200_OK;
    }
    T* p_ = nullptr;
    MemKind kind_ = MemKind::device;
    cudaStream_t s_ = nullptr;
};

// unique_ptr deleter that calls one of the library's free functions
template <auto Free>
struct FreeWith {
    template <typename T>
    void operator()(T* p) const { Free(p); }
};
// A mirror being built: freed by sprs_b200_csmat_free unless release()d into *out.
using CsmatPtr = std::unique_ptr<sprs_b200_csmat, FreeWith<sprs_b200_csmat_free>>;

// y targets of one SpMV: [0] = local y (already offset to this rank's first row), [1..n) =
// the same position inside the peer GPUs' y buffers (CUDA IPC mappings).
constexpr int SPMV_MAX_TARGETS = 8;
struct SpmvTargets {
    double* p[SPMV_MAX_TARGETS];
    int n;
};

// ---- kernels' launch wrappers (defined in the .cu files) -----------------------
// SpMV side arrays of a CSR mirror: the tile cuts, and (hot_set) the hot set where it pays
int spmv_prepare(sprs_b200_ctx* ctx, sprs_b200_csmat* m, cudaStream_t s, bool hot_set = true);
int spmv_tile_nnz();  // non-zeros per SpMV warp tile (fixed per process)
int spmv_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x, double* d_y,
                int accumulate, cudaStream_t s);
int spmv_launch_targets(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x,
                        const SpmvTargets& yt, int accumulate, cudaStream_t s);
// One chunk of the tile stream: tiles [t0, t1) + the carries of the rows ending in them; after
// chunks 0..c (in order, one stream) rows [0, tile_row[t1_c]) of y are final (spmv.cu)
int spmv_launch_tile_range(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_x,
                           double* d_y, int accumulate, uint64_t t0, uint64_t t1, cudaStream_t s);
// Chunk table of a mirror's tile stream: tiles[c] .. tiles[c+1] is chunk c, rows[c] =
// tile_row[tiles[c]] (rows [rows[c], rows[c+1]) are final once chunk c and its carries ran).
// `taper`: chunk sizes proportional to n, n-1, .., 1 (small last chunk: what follows the last
// chunk cannot overlap with compute) instead of equal.  Synchronises `s` (api.cu).
int csmat_chunk_table(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, uint64_t n_chunks, bool taper,
                      cudaStream_t s, std::vector<uint64_t>* tiles, std::vector<uint64_t>* rows);
// high-priority side stream + fork/join events of the ctx, created on first use (api.cu)
int ctx_side_stream(sprs_b200_ctx* ctx);
// copy `count` doubles at src into the same position of every buffer in dst (peer.cu)
int peer_push_launch(sprs_b200_ctx* ctx, const double* src, const SpmvTargets& dst, uint64_t count,
                     cudaStream_t s);
int spmm_rowmaj_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const double* d_b,
                       uint64_t ldb, uint64_t k, double* d_c, uint64_t ldc, int accumulate,
                       cudaStream_t s);
int triplets_to_csr_launch(sprs_b200_ctx* ctx, uint64_t rows, uint64_t cols, uint64_t n,
                           const uint32_t* d_row, const uint32_t* d_col, const double* d_val,
                           CsmatPtr* out, cudaStream_t s);
int transpose_launch(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, CsmatPtr* out, cudaStream_t s);
// CSR form of a mirror for the product kernels: the mirror itself or (CSC) its cached
// device conversion, owned by the mirror (api.cu)
int csmat_csr_view(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const sprs_b200_csmat** out);

// ---- mirrors built on the device (api.cu) -----------------------------------------
// Who holds a mirror's arrays: cudaMalloc (owned), cudaMallocAsync on the ctx stream (pooled)
// or the caller (borrowed).
enum class Arrays { owned, pooled, borrowed };
// The initialiser of every mirror: storage, shape, nnz, indptr width, who holds the arrays
sprs_b200_csmat csmat_init(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                           uint64_t nnz, int indptr_bytes, Arrays arrays);
// the same on the heap (no arrays yet)
CsmatPtr new_result(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols, uint64_t nnz,
                    int indptr_bytes, Arrays arrays);
// 4, or 8 where nnz needs it.  SPRS_B200_FORCE_INDPTR64=1 is a TEST hook: 8 always, so that
// the uint64 instantiations of the kernels run at sizes a test can afford.
int indptr_bytes_for(uint64_t nnz);
// a new mirror's indptr / indices / data, stream-ordered on s where it is pooled
int alloc_result(sprs_b200_ctx* ctx, sprs_b200_csmat* m, cudaStream_t s, const char* what);
// The finishing step of a new mirror: its SpMV partition (hot_set: and the hot set where it
// pays), then wait for s; on success m is handed out through *out.
int finish_result(sprs_b200_ctx* ctx, CsmatPtr& m, cudaStream_t s, const char* what, bool hot_set,
                  sprs_b200_csmat** out);

// ---- small device helpers -----------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// ---- progress-bounded waits on per-row ready flags (DESIGN.md 4.8), shared by the triangular
// solves (trisolve.cu) and the LDL^T factorization (ldl.cu).  Rows are claimed by a ticket
// counter in dependency order, so a wait always ends unless the whole launch stands still.
// wait_ready is a template so that only the files that wait, and so include ptx.cuh, need the
// definition of ld_acquire_u32.
static __device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p);  // ptx.cuh
constexpr long long TRI_WAIT_BOUND = 1ll << 34;  // cycles: ~9 s at 1.98 GHz

// The launch's progress: the sum of every warp's count (each only grows during a launch).
__device__ __forceinline__ unsigned long long progress_sum(const unsigned long long* w, uint64_t n) {
    unsigned long long sum = 0;
    for (uint64_t i = 0; i < n; ++i) sum += __ldcg(w + i);
    return sum;
}

// Wait until row c's flag holds `epoch`.  false: the launch's progress stood still for a whole
// TRI_WAIT_BOUND interval (read only once a wait has lasted TRI_WAIT_BOUND: no cost before).
template <typename Flag>
__device__ __forceinline__ bool wait_ready(const Flag* flag, Flag epoch,
                                           const unsigned long long* progress, uint64_t n_progress) {
    if (ld_acquire_u32(flag) == epoch) return true;
    long long start = clock64();
    bool have = false;
    unsigned long long seen = 0;
    unsigned backoff = 32;
    for (;;) {
        __nanosleep(backoff);
        if (ld_acquire_u32(flag) == epoch) return true;
        if (backoff < 1024) backoff <<= 1;
        if (clock64() - start > TRI_WAIT_BOUND) {
            const unsigned long long now = progress_sum(progress, n_progress);
            if (have && now == seen) return false;
            have = true;  // the launch moved (or this is the first look): wait on
            seen = now;
            start = clock64();
        }
    }
}
#endif

// ---- the triangular solve of trisolve.cu as a building block (ldl.cu): a plan for a
// unit-diagonal triangle stored without its diagonal (no lookup, no division, never singular).
// `csr` is borrowed and must outlive the plan; free it with sprs_b200_trisolve_free.
int trisolve_unit_plan(sprs_b200_ctx* ctx, const sprs_b200_csmat* csr, int tri,
                       sprs_b200_trisolve** out);
// enqueue one solve of d_x in place on `s` (reports an earlier wait-bound breach first)
int trisolve_enqueue(sprs_b200_trisolve* plan, double* d_x, cudaStream_t s);
// ERR_CUDA once if a solve of the plan breached the wait bound, else OK
int trisolve_check_breach(sprs_b200_trisolve* plan);
